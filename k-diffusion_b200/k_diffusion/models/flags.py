"""Backend switches (the reference's env flags live in models/flags.py:9-14) and the reference's activation checkpointing flag (:17-31).

K_DIFFUSION_USE_COMPILE / K_DIFFUSION_USE_FLASH_2 are accepted and ignored: there is no
torch.compile or flash-attn path here.  The only switch is the arithmetic of the token stream:

    KDB200_PRECISION = auto | fp32 | bf16 | tf32 | fp16      (default auto)

auto = bf16 when the call happens under torch.autocast(bfloat16) or the module's parameters are
bf16 (what `accelerate` mixed precision does for the reference), fp32 otherwise -- sample.py never
enables autocast, so the reference's inference default is true fp32 and so is ours.  tf32 (the image_v1
U-Net only, never chosen by auto): convolution and attention operands rounded to tf32 with fp32 accumulation -- what the
reference's Conv2d already computes on an H100, where torch.backends.cudnn.allow_tf32 is True by default.  fp16 (the image_v1
U-Net only, never chosen by auto, not even for fp16 parameters or under autocast(float16)): the same operands rounded to fp16 --
the 10 explicit significand bits of tf32, a narrower exponent range, twice the tensor-core rate.
"""
import os
import threading
from contextlib import contextmanager

import torch


def get_use_compile():
    return False


def get_use_flash_attention_2():
    return False


state = threading.local()
state.checkpointing = False


@contextmanager
def checkpointing(enable=True):
    """Within the block, get_checkpointing() returns `enable` on this thread (models/flags.py:17-31), which the reference's models read to
    recompute activations in their backward (torch.utils.checkpoint) instead of keeping them.  The native models ignore it: their backward
    already keeps only the residual stream entering each attention and feed-forward half on a tape and recomputes every activation from it
    (DESIGN section 3), so there is nothing more to drop."""
    try:
        old, state.checkpointing = get_checkpointing(), enable
        yield
    finally:
        state.checkpointing = old


def get_checkpointing():
    return getattr(state, "checkpointing", False)


def resolve_precision(requested, param_dtype):
    req = (requested or os.environ.get("KDB200_PRECISION", "auto")).lower()
    if req in ("fp32", "float32"):
        return "fp32"
    if req in ("bf16", "bfloat16"):
        return "bf16"
    if req == "tf32":
        return "tf32"
    if req in ("fp16", "float16"):
        return "fp16"
    if req != "auto":
        raise ValueError(f"unknown precision {req!r}")
    if param_dtype == torch.bfloat16:
        return "bf16"
    if torch.is_autocast_enabled() and torch.get_autocast_gpu_dtype() == torch.bfloat16:
        return "bf16"
    return "fp32"
