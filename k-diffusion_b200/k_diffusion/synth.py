"""Deterministic synthetic weights for benchmarks and parity tests.

A freshly constructed image_transformer_v2 outputs exactly zero (every out_proj / down_proj /
AdaRMSNorm.linear / patch_out weight is zero-initialised, reference image_transformer_v2.py:37-41,
159,365,485,706), so "random-init" timing or parity runs need every tensor filled.  The recipe
below depends only on (key name, shape, seed) -- not on module construction order or the global
RNG -- so the reference model, the oracle and the native engine can all be given bit-identical
weights without shipping a checkpoint.

This module is standalone on purpose (imports only torch/zlib): `oracle/make_golden.py` loads it by
file path next to the reference's own `k_diffusion` package.
"""
import math
import zlib

import torch

# Tensors the reference zero-initialises; filled with a small std so a 50-step solve stays well
# conditioned in fp32 (SURVEY.md section 8c: std 0.02 keeps the fp32-vs-fp64 drift below 1e-5).
_ZERO_INIT_SUFFIXES = ("out_proj.weight", "down_proj.weight", "norm.linear.weight", "patch_out.proj.weight")
ZERO_INIT_STD = 0.02


def _gen(key, seed):
    return torch.Generator().manual_seed((zlib.crc32(key.encode()) + 1000003 * int(seed)) % (2 ** 62))


def synth_tensor(key, shape, seed=0):
    """fp32 CPU tensor for state-dict entry `key` of the given shape; None = keep the constructed value."""
    g = _gen(key, seed)
    shape = tuple(shape)
    if key.endswith("pos_emb.freqs"):
        return None                                    # fixed by formula, not learned
    if key.endswith(_ZERO_INIT_SUFFIXES):
        return torch.randn(shape, generator=g) * ZERO_INIT_STD
    if key.endswith("self_attn.scale"):
        return 5.0 + 10.0 * torch.rand(shape, generator=g)          # cosine-sim temperature, init 10
    # image_transformer_v1 (reference models/image_transformer_v1.py:108-128, axial_rope.py:86-93)
    if key.endswith("qk_norm.scale"):
        return 2.5 + 2.8 * torch.rand(shape, generator=g)           # log temperature, init ln 10; above ln 100 = 4.61 is clamped
    if key.endswith(("pos_emb.freqs_h", "pos_emb.freqs_w")):
        return math.log(math.pi) + math.log(5.0) * torch.rand(shape, generator=g)   # log frequencies, init log-spaced pi .. 5 pi
    if key.endswith("fac"):
        return 0.3 + 0.4 * torch.rand(shape, generator=g)           # TokenSplit lerp factor, init 0.5
    if key.endswith(".scale"):
        return 1.0 + 0.1 * torch.randn(shape, generator=g)          # RMSNorm scale, init 1
    if key in ("time_emb.weight", "aug_emb.weight", "class_emb.weight"):
        return torch.randn(shape, generator=g)                      # FourierFeatures buffers / nn.Embedding
    # image_v1 U-Net (reference models/image_v1.py, layers.py:162-280)
    if key.endswith(".kernel") and shape == (4, 4):                 # Downsample2d / Upsample2d filter buffers
        k1 = torch.tensor([[1 / 8, 3 / 8, 3 / 8, 1 / 8]]) * (2 if ".u_blocks." in key else 1)
        return k1.T @ k1
    if key.endswith("timestep_embed.weight"):
        return torch.randn(shape, generator=g)                      # FourierFeatures buffer
    if key.endswith(("mapper.weight", "main.6.weight", "proj_out.weight")) or key.endswith(".bias"):
        return torch.randn(shape, generator=g) * ZERO_INIT_STD      # zero-initialised in the reference; biases small
    if key.endswith(".weight") and len(shape) == 4:
        return torch.randn(shape, generator=g) / math.sqrt(3.0 * math.prod(shape[1:]))
    if key.endswith(".weight") and len(shape) == 2:
        return torch.randn(shape, generator=g) / math.sqrt(3.0 * shape[1])   # variance of nn.Linear's default
    raise KeyError(f"synth_tensor: no recipe for {key} {shape}")


def synth_state_dict(shapes, seed=0, base=None):
    """`shapes`: {key: shape}.  `base`: state dict supplying values for keys the recipe leaves alone."""
    out = {}
    for key in sorted(shapes):
        t = synth_tensor(key, shapes[key], seed)
        if t is None:
            if base is None:
                raise KeyError(f"{key} needs a constructed value (pass base=model.state_dict())")
            t = base[key].detach().clone().float().cpu()
        out[key] = t
    return out


def synth_init_(module, seed=0):
    """Load the synthetic weights into any module exposing the reference state-dict layout."""
    base = module.state_dict()
    sd = synth_state_dict({k: v.shape for k, v in base.items()}, seed, base)
    module.load_state_dict({k: v.to(base[k].device, base[k].dtype) for k, v in sd.items()})
    return module
