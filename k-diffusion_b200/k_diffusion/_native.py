"""ctypes binding of libkdb200.so (C ABI declared in include/kdiffusion_b200.h).

There is deliberately NO fallback: if the shared library is missing or a tensor is not on a CUDA
device the call raises.  PyTorch is used only for device memory, streams and views.
"""
import contextlib
import copy
import ctypes
import math
import functools
import os
from pathlib import Path
from typing import NamedTuple

import torch

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("KDB200_LIB", _HERE / "_lib" / "libkdb200.so"))

PREC_FP32, PREC_BF16, PREC_TF32, PREC_FP16 = 0, 1, 2, 3
ATTN_NONE, ATTN_GLOBAL, ATTN_NEIGHBORHOOD, ATTN_SHIFTED_WINDOW = 0, 1, 2, 3
FAMILY_ITV2, FAMILY_ITV1 = 0, 1
MAX_LEVELS = 8
ABI_VERSION = 28

_vp, _i32, _i64, _f32, _f64, _u64, _sz = (ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double,
                                           ctypes.c_uint64, ctypes.c_size_t)


class KdbModelConfig(ctypes.Structure):
    _fields_ = [
        ("n_levels", _i32), ("in_channels", _i32), ("out_channels", _i32), ("patch_h", _i32), ("patch_w", _i32),
        ("mapping_width", _i32), ("mapping_depth", _i32), ("mapping_d_ff", _i32), ("num_classes", _i32), ("mapping_cond_dim", _i32),
        ("width", _i32 * MAX_LEVELS), ("depth", _i32 * MAX_LEVELS), ("d_ff", _i32 * MAX_LEVELS), ("attn_type", _i32 * MAX_LEVELS),
        ("d_head", _i32 * MAX_LEVELS), ("attn_param", _i32 * MAX_LEVELS), ("family", _i32),
    ]


class KdbUNetConfig(ctypes.Structure):
    _fields_ = [
        ("n_levels", _i32), ("in_channels", _i32), ("patch_size", _i32), ("mapping_out", _i32), ("mapping_cond_dim", _i32),
        ("augment_wrapper", _i32), ("skip_stages", _i32), ("has_variance", _i32),
        ("depth", _i32 * MAX_LEVELS), ("channels", _i32 * MAX_LEVELS), ("self_attn", _i32 * MAX_LEVELS),
    ]


EMA_LERP, EMA_COPY = 0, 1


class KdbEmaSeg(ctypes.Structure):
    _fields_ = [("src", _vp), ("dst", _vp), ("n", _i64), ("mode", _i32)]


# name -> (restype, argtypes); this table is also what tests/test_abi.py checks against the header.
SIGNATURES = {
    "kdb_abi_version": (_i32, []),
    "kdb_last_error": (ctypes.c_char_p, []),
    "kdb_launch_count": (_u64, []),
    "kdb_launch_breakdown": (_i32, [ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(_u64), _i32]),
    "kdb_profile_begin": (_i32, [_i32, _vp]),
    "kdb_profile_end": (_i32, [ctypes.POINTER(_i32), ctypes.POINTER(_f32), _i32]),
    "kdb_profile_gate": (_i32, [_i64, _vp]),
    "kdb_solver_euler_step": (_i32, [_vp, _vp, _vp, _vp, _i64, _f32, _f32, _vp]),
    "kdb_solver_heun_correct": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _f32, _f32, _vp]),
    "kdb_solver_dpmpp_2m_step": (_i32, [_vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _vp]),
    "kdb_solver_lincomb": (_i32, [ctypes.POINTER(_vp), ctypes.POINTER(_f32), _i32, _vp, _i64, _vp]),
    "kdb_solver_cfg_combine": (_i32, [_vp, _vp, _vp, _i64, _f32, _vp]),
    "kdb_solver_dpm_error": (_i32, [_vp, _vp, _vp, _i64, _f32, _f32, _vp, _vp]),
    "kdb_solver_rk_error": (_i32, [_vp, _vp, _vp, _i64, _f32, _f32, _vp, _vp]),
    "kdb_solver_to_d": (_i32, [_vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "kdb_precond_scale_in": (_i32, [_vp, _vp, _f32, _vp, _i32, _i64, _vp]),
    "kdb_precond_combine": (_i32, [_vp, _vp, _vp, _f32, _vp, _i32, _i64, _vp]),
    "kdb_external_scale_in": (_i32, [_vp, _vp, _f32, _vp, _i32, _i64, _vp]),
    "kdb_external_combine": (_i32, [_i32, _vp, _i32, _i64, _vp, _vp, _f32, _vp, _i32, _i64, _vp]),
    "kdb_noise_normal": (_i32, [_vp, _vp, _u64, _i32, _i64, _vp]),
    "kdb_noise_brownian": (_i32, [_vp, _vp, _i32, _i64, _f64, _f64, _f64, _f64, _i32, _vp]),
    "kdb_model_create": (_i32, [ctypes.POINTER(KdbModelConfig), ctypes.POINTER(_vp)]),
    "kdb_model_destroy": (None, [_vp]),
    "kdb_model_set_tensor": (_i32, [_vp, ctypes.c_char_p, _vp, ctypes.POINTER(_i64), _i32]),
    "kdb_model_finalize": (_i32, [_vp, _vp]),
    "kdb_model_cond_stride": (_i64, [_vp]),
    "kdb_model_conditioning": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "kdb_model_workspace_bytes": (_sz, [_vp, _i32, _i32, _i32, _i32]),
    "kdb_model_forward": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _sz, _vp]),
    "kdb_model_forward_jvp": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "kdb_model_vjp_workspace_bytes": (_i64, [_vp, _i32, _i32, _i32]),
    "kdb_model_forward_vjp": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "kdb_model_set_grad": (_i32, [_vp, ctypes.c_char_p, _vp, ctypes.POINTER(_i64), _i32]),
    "kdb_model_train_workspace_bytes": (_i64, [_vp, _i32, _i32, _i32]),
    "kdb_model_forward_train": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "kdb_model_train_forward": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _sz, _vp]),
    "kdb_loss_noised_input": (_i32, [_vp, _vp, _vp, _f32, _vp, _i32, _i64, _vp]),
    "kdb_denoiser_loss": (_i32, [_i32, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _i32, _i64, _vp]),
    "kdb_variance_loss": (_i32, [_vp, _vp, _vp, _f32, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "kdb_model_debug_tap": (_i32, [_vp, ctypes.c_char_p, _vp, _i64]),
    "kdb_model_tap_count": (_i64, [_vp]),
    "kdb_unet_create": (_i32, [ctypes.POINTER(KdbUNetConfig), ctypes.POINTER(_vp)]),
    "kdb_unet_destroy": (_i32, [_vp]),
    "kdb_unet_set_tensor": (_i32, [_vp, ctypes.c_char_p, _vp, ctypes.POINTER(_i64), _i32]),
    "kdb_unet_finalize": (_i32, [_vp, _vp]),
    "kdb_unet_cond_stride": (_i64, [_vp]),
    "kdb_unet_conditioning": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "kdb_unet_workspace_bytes": (_i64, [_vp, _i32, _i32, _i32, _i32]),
    "kdb_unet_forward": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _sz, _vp]),
    "kdb_unet_forward_variance": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "kdb_unet_debug_tap": (_i32, [_vp, ctypes.c_char_p, _vp, _i64]),
    "kdb_unet_tap_count": (_i64, [_vp]),
    "kdb_unet_set_grad": (_i32, [_vp, ctypes.c_char_p, _vp, ctypes.POINTER(_i64), _i32]),
    "kdb_unet_train_workspace_bytes": (_i64, [_vp, _i32, _i32, _i32]),
    "kdb_unet_forward_train": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "kdb_unet_forward_train_variance": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "kdb_unet_conv_wgrad": (_i32, [_vp, _i32, _vp, _i32, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "kdb_unet_adagn_vjp": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _i64, _i32, _i32, _i32, _i32, _vp]),
    "kdb_unet_flip_conv_weight": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp]),
    "kdb_unet_resample_vjp": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_unet_mapping_vjp": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "kdb_unet_proj_out_vjp": (_i32, [_vp, _vp, _vp, _i64, _i32, _i32, _vp]),
    "kdb_unet_unshuffle": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_wgrad": (_i32, [_i32, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "kdb_wgrad_patch_in": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "kdb_wgrad_patch_out": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "kdb_norm_scale_grad": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i64, _i64, _i32, _vp, _vp]),
    "kdb_colsum": (_i32, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "kdb_split_fac_grad": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "kdb_class_emb_grad": (_i32, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, _vp]),
    "kdb_gemm_vjp": (_i32, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_rmsnorm_vjp": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp]),
    "kdb_qknorm_rope_vjp": (_i32, [_vp, _vp, _vp, _vp, _vp, _f32, _i32, _i64, _i32, _i32, _i32, _vp, _vp]),
    "kdb_geglu_vjp": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp]),
    "kdb_split_vjp_gather": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "kdb_split_unpatch_lerp": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "kdb_merge_scatter_add": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "kdb_patch_out_vjp": (_i32, [_vp, _vp, _vp, _vp, _vp, _f32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "kdb_patch_in_vjp": (_i32, [_vp, _vp, _vp, _vp, _f32, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_model_mapping_vjp": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "kdb_gemm_bf16": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "kdb_gemm_bf16_geglu": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "kdb_ffn_fused_bf16": (_i32, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "kdb_attn_block_bf16": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "kdb_attention": (_i32, [_i32, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "kdb_attention_jvp": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_attention_vjp": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_unet_conv": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_unet_conv_tf32": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_unet_conv_fp16": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "kdb_mmd_workspace_bytes": (_i64, [ctypes.POINTER(_i64), ctypes.POINTER(_i64), _i32]),
    "kdb_mmd_sums": (_i32, [_vp, _i64, _vp, _i64, _i32, ctypes.POINTER(_i64), ctypes.POINTER(_i64), _i32, _vp, _vp, _sz, _vp]),
    "kdb_polynomial_kernel": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "kdb_feature_mean_cov": (_i32, [_vp, _i64, _i32, _vp, _vp, _vp]),
    "kdb_ema_update": (_i32, [ctypes.POINTER(KdbEmaSeg), _i32, _f32, _vp]),
    "kdb_augment": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, ctypes.c_double, ctypes.c_double, ctypes.c_double, _i32, _vp, _vp, _vp,
                           _vp, _vp]),
}

_lib = None


class NativeLibraryError(RuntimeError):
    pass


def lib():
    """Load libkdb200.so once.  Raises loudly when it has not been built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise NativeLibraryError(
                f"{LIB_PATH} not found: build it with `python __graft_entry__.py` (or `make -C k-diffusion_b200/csrc`). "
                "This package has no CPU or eager fallback.")
        handle = ctypes.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        got = handle.kdb_abi_version()
        if got != ABI_VERSION:
            raise NativeLibraryError(f"{LIB_PATH}: ABI version {got}, binding expects {ABI_VERSION}; rebuild")
        _lib = handle
    return _lib


def check(rc):
    if rc != 0:
        msg = lib().kdb_last_error().decode(errors="replace")
        if rc == -1:
            raise ValueError(msg)
        raise RuntimeError(f"libkdb200 error {rc}: {msg}")


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("k_diffusion (H100-native) operates on CUDA tensors only; there is no CPU fallback "
                               f"(got a {t.device} tensor)")


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


_NULL_CTX = contextlib.nullcontext()


def device_of(t):
    """Context that makes `t`'s GPU the current device (kernels launch on the CURRENT device's current stream and the engine
    allocates there).  A no-op object when it already is -- the common case costs one integer compare."""
    if t is None or not t.is_cuda or t.device.index == torch.cuda.current_device():
        return _NULL_CTX
    return torch.cuda.device(t.device)


def _on_device_of_first(fn):
    """Run a kernel wrapper on the device of its first tensor argument (a list of tensors counts by its first entry)."""
    @functools.wraps(fn)
    def wrapper(first, *args, **kwargs):
        t = first[0] if isinstance(first, (list, tuple)) else first
        ctx = device_of(t)
        if ctx is _NULL_CTX:
            return fn(first, *args, **kwargs)
        with ctx:
            return fn(first, *args, **kwargs)
    return wrapper


def f32c(t):
    """fp32 contiguous view/copy (torch plumbing)."""
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def launch_count():
    return int(lib().kdb_launch_count())


def launch_breakdown():
    n = lib().kdb_launch_breakdown(None, None, 0)
    names = (ctypes.c_char_p * n)()
    counts = (_u64 * n)()
    lib().kdb_launch_breakdown(names, counts, n)
    return {names[i].decode(): int(counts[i]) for i in range(n)}


class profile:
    """with profile() as p: ...  -> p.by_family = {family: (launches, total_ms)}, p.launches = [(family, ms)]

    gate_ms > 0 first parks the stream for that long (kdb_profile_gate) so the host can enqueue the region's launches ahead of
    the GPU: the kernels then run back to back and the event intervals hold no host launch gaps (what a graph replay sees)."""

    def __init__(self, max_launches=200000, gate_ms=0.0):
        self.cap, self.gate_ms = max_launches, gate_ms

    def __enter__(self):
        if self.gate_ms > 0:
            check(lib().kdb_profile_gate(int(self.gate_ms * 1e6), stream()))
        check(lib().kdb_profile_begin(self.cap, stream()))
        return self

    def __exit__(self, *exc):
        fam = (_i32 * self.cap)()
        ms = (_f32 * self.cap)()
        n = lib().kdb_profile_end(fam, ms, self.cap)
        names = list(launch_breakdown())
        self.launches = [(names[fam[i]], float(ms[i])) for i in range(min(n, self.cap))]
        self.by_family = {}
        for f, t in self.launches:
            c, tot = self.by_family.get(f, (0, 0.0))
            self.by_family[f] = (c + 1, tot + t)
        return False


# ---------------------------------------------------------------------------------------------
# solver elementwise ops
# ---------------------------------------------------------------------------------------------

def _out_like(x, out):
    return torch.empty_like(x) if out is None else out


@_on_device_of_first
def euler_step(x, den, r, noise=None, cn=0.0, out=None):
    """x + (x - den) * r [+ noise * cn]"""
    require_cuda(x, den, noise)
    out = _out_like(x, out)
    check(lib().kdb_solver_euler_step(ptr(x), ptr(den), ptr(noise), ptr(out), x.numel(), r, cn, stream()))
    return out


@_on_device_of_first
def heun_correct(x, den1, x2, den2, a1, a2, out=None):
    """x + (x - den1) * a1 + (x2 - den2) * a2"""
    require_cuda(x, den1, x2, den2)
    out = _out_like(x, out)
    check(lib().kdb_solver_heun_correct(ptr(x), ptr(den1), ptr(x2), ptr(den2), ptr(out), x.numel(), a1, a2, stream()))
    return out


@_on_device_of_first
def dpmpp_2m_step(x, den, old_den, a, b, k1, k0, out=None):
    """a x - b (k1 den + k0 old_den)"""
    require_cuda(x, den, old_den)
    out = _out_like(x, out)
    check(lib().kdb_solver_dpmpp_2m_step(ptr(x), ptr(den), ptr(old_den), ptr(out), x.numel(), a, b, k1, k0, stream()))
    return out


@_on_device_of_first
def lincomb(tensors, coefs, out=None):
    """sum_i coefs[i] * tensors[i]   (1..6 fp32 tensors of equal size)"""
    require_cuda(*tensors)
    n = len(tensors)
    out = _out_like(tensors[0], out)
    ptrs = (_vp * n)(*[t.data_ptr() for t in tensors])
    cs = (_f32 * n)(*[float(c) for c in coefs])
    check(lib().kdb_solver_lincomb(ptrs, cs, n, ptr(out), tensors[0].numel(), stream()))
    return out


@_on_device_of_first
def cfg_combine(uncond, cond, scale, out=None):
    """uncond + (cond - uncond) * scale"""
    require_cuda(uncond, cond)
    out = _out_like(uncond, out)
    check(lib().kdb_solver_cfg_combine(ptr(uncond), ptr(cond), ptr(out), uncond.numel(), float(scale), stream()))
    return out


@_on_device_of_first
def dpm_error(x_low, x_high, x_prev, atol, rtol):
    """||(x_low - x_high) / max(atol, rtol * max(|x_low|, |x_prev|))||_2 / sqrt(numel) as a Python float (one device->host read: the adaptive
    DPM-Solver decides accept / reject on the host, sampling.py:466-470 of the reference)."""
    require_cuda(x_low, x_high, x_prev)
    scratch = torch.empty(512, dtype=torch.float32, device=x_low.device)
    check(lib().kdb_solver_dpm_error(ptr(f32c(x_low)), ptr(f32c(x_high)), ptr(f32c(x_prev)), x_low.numel(), float(atol), float(rtol), ptr(scratch), stream()))
    return math.sqrt(float(scratch[0])) / math.sqrt(x_low.numel())


@_on_device_of_first
def rk_error(err, y0, y1, atol, rtol):
    """||err / (atol + rtol * max(|y0|, |y1|))||_2 / sqrt(numel) as a Python float: the error ratio of one embedded Runge-Kutta step
    (the dopri5 integration of log_likelihood, reference sampling.py:298)."""
    require_cuda(err, y0, y1)
    scratch = torch.empty(512, dtype=torch.float32, device=err.device)
    check(lib().kdb_solver_rk_error(ptr(f32c(err)), ptr(f32c(y0)), ptr(f32c(y1)), err.numel(), float(atol), float(rtol), ptr(scratch), stream()))
    return math.sqrt(float(scratch[0])) / math.sqrt(err.numel())


@_on_device_of_first
def to_d(x, den, sigma_b, out=None):
    """(x - den) / sigma[b]"""
    require_cuda(x, den, sigma_b)
    out = _out_like(x, out)
    check(lib().kdb_solver_to_d(ptr(x), ptr(den), ptr(sigma_b), ptr(out), x.shape[0], x[0].numel(), stream()))
    return out


@_on_device_of_first
def precond_scale_in(x, sigma, sigma_data, out=None):
    require_cuda(x, sigma)
    out = _out_like(x, out)
    check(lib().kdb_precond_scale_in(ptr(x), ptr(sigma), sigma_data, ptr(out), x.shape[0], x[0].numel(), stream()))
    return out


@_on_device_of_first
def precond_combine(f, x, sigma, sigma_data, out=None):
    require_cuda(f, x, sigma)
    out = _out_like(x, out)
    check(lib().kdb_precond_combine(ptr(f), ptr(x), ptr(sigma), sigma_data, ptr(out), x.shape[0], x[0].numel(), stream()))
    return out


EXTERNAL_EPS, EXTERNAL_V = 0, 1
_EXT_DTYPE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


@_on_device_of_first
def external_scale_in(x, sigma, sigma_data=1.0):
    """x [B, ...] fp32 contiguous, sigma [B] fp32 -> x * c_in, c_in = 1 / sqrt(sigma^2 + sigma_data^2) rounded as the reference's
    torch expression (external.py get_scalings)."""
    require_cuda(x, sigma)
    out = torch.empty_like(x)
    B = x.shape[0]
    check(lib().kdb_external_scale_in(ptr(x), ptr(sigma), float(sigma_data), ptr(out), B, x.numel() // B, stream()))
    return out


LOSS_DENOISER, LOSS_SIMPLE = 0, 1
LOSS_VARIANCE = 2     # DenoiserWithVariance.loss: kdb_variance_loss on the model's F and logvar (no kdb_denoiser_loss kind)


@_on_device_of_first
def loss_noised_input(x, noise, sigma, sigma_data):
    """(x + noise * sigma) * c_in(sigma): the inner model's input of a training loss (layers.py:79-81)"""
    require_cuda(x, noise, sigma)
    out = torch.empty_like(x)
    check(lib().kdb_loss_noised_input(ptr(x), ptr(noise), ptr(sigma), float(sigma_data), ptr(out), x.shape[0], x[0].numel(), stream()))
    return out


@_on_device_of_first
def denoiser_loss(x, noise, sigma, weight, sigma_data, f, kind):
    """-> (loss [B], d loss[b] / d f): kdb_denoiser_loss (LOSS_DENOISER: layers.py:76-86 with scales == 1; LOSS_SIMPLE: :107-111)"""
    require_cuda(x, noise, sigma, weight, f)
    loss = torch.empty(x.shape[0], device=x.device, dtype=torch.float32)
    cot = torch.empty_like(f)
    check(lib().kdb_denoiser_loss(kind, ptr(x), ptr(noise), ptr(sigma), ptr(weight), float(sigma_data), ptr(f), ptr(loss), ptr(cot),
                                  x.shape[0], x[0].numel(), stream()))
    return loss, cot


@_on_device_of_first
def variance_loss(x, noise, sigma, sigma_data, f, logvar):
    """-> (loss [B], d loss[b] / d f, d loss[b] / d logvar[b]): kdb_variance_loss (layers.py:93-101)"""
    require_cuda(x, noise, sigma, f, logvar)
    B = x.shape[0]
    loss, dlogvar = (torch.empty(B, device=x.device, dtype=torch.float32) for _ in range(2))
    cot = torch.empty_like(f)
    check(lib().kdb_variance_loss(ptr(x), ptr(noise), ptr(sigma), float(sigma_data), ptr(f), ptr(logvar), ptr(loss), ptr(cot), ptr(dlogvar), B,
                                  x[0].numel(), stream()))
    return loss, cot, dlogvar


def _per_sample_stride(f, B):
    """f's batch stride if each of its B samples is one contiguous run (a contiguous tensor, or a channel slice of one such as the
    eps half of a learned-variance output), else None."""
    shape, strides = f.shape, f.stride()
    if f.ndim == 0 or shape[0] != B:
        return None
    run = 1
    for d in range(f.ndim - 1, 0, -1):
        if shape[d] != 1 and strides[d] != run:
            return None
        run *= shape[d]
    return strides[0] if B > 1 else run


def external_combine(kind, f, x, sigma, sigma_data=1.0):
    """The output combine of an external wrapper: kind EXTERNAL_EPS -> x + f * (-sigma), EXTERNAL_V -> f * c_out + x * c_skip.
    f (the inner model's output: fp32, fp16 or bf16, each sample contiguous, any batch stride) is read in place; either f or x
    may be None, which drops its term.  x fp32 contiguous, sigma [B] fp32 -> fp32 [B, ...] of x's (or f's) shape."""
    require_cuda(f, x, sigma)
    like = x if x is not None else f
    B = like.shape[0]
    n = like.numel() // B
    stride, code = 0, 0
    if f is not None:
        if f.dtype not in _EXT_DTYPE:
            raise TypeError(f"the inner model returned {f.dtype}; the external wrappers take fp32, fp16 or bf16 outputs")
        if x is not None and f.shape != x.shape:
            raise ValueError(f"inner model output of shape {tuple(f.shape)} for an input of shape {tuple(x.shape)}")
        stride = _per_sample_stride(f, B)
        if stride is None:
            f = f.contiguous()
            stride = n
        code = _EXT_DTYPE[f.dtype]
    out = torch.empty(like.shape, dtype=torch.float32, device=like.device)
    with device_of(like):
        check(lib().kdb_external_combine(kind, ptr(f), code, stride, ptr(x), ptr(sigma), float(sigma_data), ptr(out), B, n, stream()))
    return out


@_on_device_of_first
def noise_normal(like, seeds, stream_id, out=None):
    require_cuda(like, seeds)
    out = _out_like(like, out)
    check(lib().kdb_noise_normal(ptr(out), ptr(seeds), int(stream_id) & (2 ** 64 - 1), like.shape[0], like[0].numel(), stream()))
    return out


@_on_device_of_first
def noise_brownian(like, seeds, t_min, t_max, t0, t1, depth=24, out=None):
    require_cuda(like, seeds)
    out = _out_like(like, out)
    check(lib().kdb_noise_brownian(ptr(out), ptr(seeds), like.shape[0], like[0].numel(), t_min, t_max, t0, t1, depth, stream()))
    return out


# ---------------------------------------------------------------------------------------------
# model engine
# ---------------------------------------------------------------------------------------------

_ATTN_CODE = {"none": ATTN_NONE, "global": ATTN_GLOBAL, "neighborhood": ATTN_NEIGHBORHOOD, "shifted-window": ATTN_SHIFTED_WINDOW}


UNET_NO_DERIVATIVE = "the image_v1 U-Net engine has no derivative: only its forward is built (no JVP, VJP or autograd through x)"


def unet_has_no_derivative(*args, **kwargs):
    """What every derivative entry point of the U-Net does (the engine, the model and the augment wrapper around it)."""
    raise NotImplementedError(UNET_NO_DERIVATIVE)


def check_input(x, sigma, dropout):
    """The checks of x and sigma every native model makes before evaluating; `dropout`: the model is in training mode with dropout."""
    require_cuda(x, sigma)
    if x.ndim != 4:
        raise ValueError(f"expected x of shape [B, C, H, W], got {tuple(x.shape)}")
    if dropout:
        raise RuntimeError("dropout > 0 in training mode: the native path is inference only -- call model.eval()")


def require_cond(class_cond, mapping_cond, class_needed, mapping_needed):
    """The native front ends' refusal of a missing conditioning input the model needs (the reference's forwards raise the same)."""
    if class_cond is None and class_needed:
        raise ValueError("class_cond must be specified if num_classes > 0")
    if mapping_cond is None and mapping_needed:
        raise ValueError("mapping_cond must be specified if mapping_cond_dim > 0")


class Evaluation:
    """The answer of a native model's front end `native_eval(x, sigma, aug_cond, class_cond, mapping_cond, precision)`, which validates
    those inputs: the bound engine, the precision code, x as fp32, sigma as [B] fp32 (None when the caller brings its own rows, as the
    sampler does) and the conditioning exactly as the engine takes it (`takes_class` / `takes_mapping`: whether it takes class_cond /
    mapping_cond; aug_cond is always taken)."""

    def __init__(self, engine, precision, x, sigma, aug_cond, class_cond, mapping_cond, takes_class, takes_mapping):
        self.engine, self.precision, self.dtype = engine, precision, x.dtype
        self.x = f32c(x)
        self.sigma = None
        if sigma is not None:
            self.sigma = f32c(sigma).expand(x.shape[0]).contiguous() if sigma.numel() == 1 else f32c(sigma)
            if self.sigma.shape != (x.shape[0],):
                raise ValueError(f"sigma must have shape [{x.shape[0]}], got {tuple(sigma.shape)}")
        self._takes, self._uncond = (takes_class, takes_mapping), None
        self.cond = self.cond_args(1, aug_cond, class_cond, mapping_cond)

    def guide(self, uncond):
        """Make this the evaluation of classifier-free guidance's doubled batch [uncond | cond]: class_cond rows of class `uncond` first."""
        n = int(self.engine.cfg.num_classes)
        if self._takes[0] and not torch.cuda.is_current_stream_capturing() and not 0 <= uncond < n:
            raise IndexError(f"CFG unconditional class {uncond} outside class_emb ({n} rows)")
        self._uncond = uncond
        return self

    def cond_args(self, reps=1, aug_cond=None, class_cond=None, mapping_cond=None):
        """(aug_cond, class_cond, mapping_cond) as the engine takes them, None where it takes none, for `reps` evaluations stacked along
        the batch.  The sampler passes its own copies of the inputs this evaluation was made with (a captured graph reads static ones)."""
        class_cond = class_cond if self._takes[0] else None
        if self._uncond is not None:
            class_cond = torch.cat([torch.full_like(class_cond, self._uncond), class_cond])
        args = (aug_cond, class_cond, mapping_cond if self._takes[1] else None)
        return args if reps == 1 else tuple(None if t is None else t.repeat(reps, *([1] * (t.ndim - 1))) for t in args)

    def conditioning(self):
        return self.engine.conditioning(self.sigma, *self.cond)

    def cast(self, res):
        """An engine result (or a tuple of them) in x's dtype."""
        if self.dtype == torch.float32:
            return res
        return tuple(r.to(self.dtype) for r in res) if isinstance(res, tuple) else res.to(self.dtype)

    def forward(self, sigma_data, out=None):
        """The raw model (sigma_data 0) or the Karras-preconditioned denoiser at this evaluation's precision, in x's dtype."""
        return self.cast(self.engine.forward(self.x, self.sigma, self.conditioning(), self.engine.cond_stride, sigma_data, self.precision,
                                             out=out))


class EngineCache:
    """Base of the model classes that keep their native engines in self._engines ({key: Engine}).  An engine holds device pointers into
    the model's own tensors, so a pickled or deep-copied model starts without engines and builds its own on first use."""

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_engines"] = {}
        return state

    def __deepcopy__(self, memo):
        engines, self._engines = self._engines, {}
        try:
            new = self.__class__.__new__(self.__class__)
            memo[id(self)] = new
            new.__dict__ = copy.deepcopy(self.__dict__, memo)
        finally:
            self._engines = engines
        return new


class Engine:
    """Owns one native model handle on one device: a KdbModel for an ImageTransformerDenoiserModelV2 or V1 (`_api` "model"), or, in the
    UNetEngine subclass, a KdbUNet for an ImageDenoiserModelV1 (`_api` "unet").  Both handles take the same calls (create, destroy,
    set_tensor, finalize, cond_stride, workspace_bytes, forward, set_grad, train_workspace_bytes, debug_tap, tap_count) under kdb_<api>_*."""

    _api = "model"

    def _fn(self, name):
        return getattr(lib(), f"kdb_{self._api}_{name}")

    def __init__(self, spec):
        self.cfg = self._config(spec)
        self._h = _vp()
        check(self._fn("create")(ctypes.byref(self.cfg), ctypes.byref(self._h)))
        self._sig, self._held, self._ws, self._stride, self.device = None, {}, None, None, None
        self._grad_keys = set()

    @staticmethod
    def _config(spec):
        cfg = KdbModelConfig()
        levels = spec["levels"]
        if len(levels) > MAX_LEVELS:
            raise ValueError(f"at most {MAX_LEVELS} levels supported")
        cfg.n_levels = len(levels)
        cfg.in_channels, cfg.out_channels = spec["in_channels"], spec["out_channels"]
        cfg.patch_h, cfg.patch_w = spec["patch_size"]
        cfg.mapping_width, cfg.mapping_depth, cfg.mapping_d_ff = spec["mapping_width"], spec["mapping_depth"], spec["mapping_d_ff"]
        cfg.num_classes, cfg.mapping_cond_dim = spec["num_classes"], spec["mapping_cond_dim"]
        cfg.family = spec.get("family", FAMILY_ITV2)
        for i, lv in enumerate(levels):
            cfg.width[i], cfg.depth[i], cfg.d_ff[i] = lv["width"], lv["depth"], lv["d_ff"]
            cfg.attn_type[i] = _ATTN_CODE[lv["attn"]]
            cfg.d_head[i] = lv.get("d_head", 0)
            cfg.attn_param[i] = lv.get("attn_param", 0)
        return cfg

    def _out_channels(self, x):
        return self.cfg.out_channels

    def __del__(self):
        try:
            if getattr(self, "_h", None) and _lib is not None:
                getattr(_lib, f"kdb_{self._api}_destroy")(self._h)
                self._h = None
        except Exception:
            pass

    def bind(self, tensors):
        """tensors: {state-dict key: tensor on a CUDA device}.  Rebinds + finalizes only when something changed."""
        sig = tuple((k, t.data_ptr(), t._version, t.dtype, str(t.device)) for k, t in tensors.items())
        if sig == self._sig:
            return
        require_cuda(*tensors.values())
        devs = {t.device for t in tensors.values()}
        if len(devs) != 1:
            raise RuntimeError(f"model tensors live on several devices: {devs}")
        self.device = devs.pop()
        held = {}
        with torch.cuda.device(self.device):
            for k, t in tensors.items():
                t32 = f32c(t.detach())
                held[k] = t32
                shape = (_i64 * t32.ndim)(*t32.shape)
                check(self._fn("set_tensor")(self._h, k.encode(), ptr(t32), shape, t32.ndim))
            check(self._fn("finalize")(self._h, stream()))
        self._held = held
        self._sig = sig
        self._stride = int(self._fn("cond_stride")(self._h))

    @property
    def cond_stride(self):
        return self._stride

    def conditioning(self, sigma, aug_cond=None, class_cond=None, mapping_cond=None):
        """-> [rows, cond_stride] fp32 table (mapping network + every AdaRMSNorm projection)."""
        require_cuda(sigma, aug_cond, class_cond, mapping_cond)
        sigma = f32c(sigma)
        rows = sigma.numel()
        aug_cond = None if aug_cond is None else f32c(aug_cond)
        mapping_cond = None if mapping_cond is None else f32c(mapping_cond)
        class_cond = None if class_cond is None else class_cond.to(torch.int64).contiguous()
        out = torch.empty(rows, self._stride, device=sigma.device, dtype=torch.float32)
        with device_of(sigma):
            check(lib().kdb_model_conditioning(self._h, rows, ptr(sigma), ptr(aug_cond), ptr(class_cond), ptr(mapping_cond), ptr(out), stream()))
        return out

    def check_class_range(self, class_cond):
        """nn.Embedding raises on an out-of-range index (reference image_transformer_v2.py:735); the conditioning kernel indexes
        class_emb with it, so validate on the host (one device->host sync; callers do it once per sampler call, not per step)."""
        n = int(self.cfg.num_classes)
        if class_cond is None or n <= 0:
            return
        lo, hi = int(class_cond.min()), int(class_cond.max())
        if lo < 0 or hi >= n:
            raise IndexError(f"class_cond values must lie in [0, {n}) (class_emb has {n} rows), got [{lo}, {hi}]")

    def workspace_bytes(self, precision, B, H, W):
        """kdb_<api>_workspace_bytes: the workspace of a forward of B images"""
        need = int(self._fn("workspace_bytes")(self._h, precision, B, H, W))
        if need < 0:
            check(need)
        return need

    def _workspace(self, precision, B, H, W, device):
        return self._reserve(self.workspace_bytes(precision, B, H, W), device)

    def _reserve(self, need, device):
        """The engine's workspace of at least `need` bytes on `device`, grown and reused across calls."""
        need = int(need)
        if need < 0:
            check(need)
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=device)
        return self._ws

    def forward(self, x, sigma, cond, cond_batch_stride, sigma_data, precision, out=None):
        """x [B,C,H,W] fp32; sigma [B]; cond rows; sigma_data <= 0 -> raw inner model."""
        B, _, H, W = x.shape
        if out is None:
            out = torch.empty(B, self._out_channels(x), H, W, device=x.device, dtype=torch.float32)
        ws = self._workspace(precision, B, H, W, x.device)
        with device_of(x):
            check(self._fn("forward")(self._h, precision, B, H, W, ptr(x), ptr(sigma), float(sigma_data), ptr(cond), cond_batch_stride,
                                      ptr(out), ptr(ws), ws.numel(), stream()))
        return out

    def forward_jvp(self, x, v, sigma, cond, cond_batch_stride, sigma_data, out=None, out_tangent=None):
        """Forward-mode derivative on the fp32 path: -> (out, tangent), out as forward() at fp32, tangent = J(x) v.
        x, v [B,C,H,W] fp32 contiguous; the workspace holds 2B images (the tangent rides as the second half of the batch)."""
        B, _, H, W = x.shape
        if v.shape != x.shape:
            raise ValueError(f"tangent shape {tuple(v.shape)} != x shape {tuple(x.shape)}")
        shape = (B, self.cfg.out_channels, H, W)
        out = torch.empty(shape, device=x.device, dtype=torch.float32) if out is None else out
        out_tangent = torch.empty(shape, device=x.device, dtype=torch.float32) if out_tangent is None else out_tangent
        ws = self._workspace(PREC_FP32, 2 * B, H, W, x.device)
        with device_of(x):
            check(lib().kdb_model_forward_jvp(self._h, PREC_FP32, B, H, W, ptr(x), ptr(v), ptr(sigma), float(sigma_data), ptr(cond),
                                              cond_batch_stride, ptr(out), ptr(out_tangent), ptr(ws), ws.numel(), stream()))
        return out, out_tangent

    def forward_vjp(self, x, u, sigma, cond, cond_batch_stride, sigma_data, out=None, out_grad=None):
        """Reverse-mode derivative on the fp32 path: -> (out, grad_x), out as forward() at fp32, grad_x = u^T J(x).
        x [B,C_in,H,W] and u [B,C_out,H,W] fp32 contiguous; the workspace holds the forward's tape (kdb_model_vjp_workspace_bytes)."""
        B, _, H, W = x.shape
        shape = (B, self.cfg.out_channels, H, W)
        if tuple(u.shape) != shape:
            raise ValueError(f"cotangent shape {tuple(u.shape)} != output shape {shape}")
        out = torch.empty(shape, device=x.device, dtype=torch.float32) if out is None else out
        out_grad = torch.empty_like(x) if out_grad is None else out_grad
        ws = self._reserve(lib().kdb_model_vjp_workspace_bytes(self._h, B, H, W), x.device)
        with device_of(x):
            check(lib().kdb_model_forward_vjp(self._h, PREC_FP32, B, H, W, ptr(x), ptr(sigma), float(sigma_data), ptr(cond), cond_batch_stride,
                                              ptr(u), ptr(out), ptr(out_grad), ptr(ws), ws.numel(), stream()))
        return out, out_grad

    def train_workspace(self, B, H, W):
        """kdb_<api>_train_workspace_bytes: the workspace of forward_train for B images"""
        need = int(self._fn("train_workspace_bytes")(self._h, B, H, W))
        if need < 0:
            check(need)
        return need

    def set_grad(self, grads):
        """Binds `grads` ({state-dict key: fp32 CUDA tensor of the parameter's shape}) and unbinds every other key bound before."""
        for k in self._grad_keys - set(grads):
            check(self._fn("set_grad")(self._h, k.encode(), None, None, 0))
        for k, g in grads.items():
            dims = (_i64 * g.ndim)(*g.shape)
            check(self._fn("set_grad")(self._h, k.encode(), ptr(g), dims, g.ndim))
        self._grad_keys = set(grads)

    def forward_train(self, x, u, sigma, aug_cond, class_cond, mapping_cond, cond, grads, out=None, grad_x=None, precision=PREC_FP32):
        """Parameter gradients at the training precision (PREC_FP32 or PREC_TF32): binds `grads` ({state-dict key: fp32 CUDA tensor of the
        parameter's shape}, every other key unbound), then one kdb_model_forward_train: out = F(x), every bound gradient = u^T dF/dparam,
        grad_x (if given) u^T dF/dx."""
        B, _, H, W = x.shape
        shape = (B, self.cfg.out_channels, H, W)
        if tuple(u.shape) != shape:
            raise ValueError(f"cotangent shape {tuple(u.shape)} != output shape {shape}")
        out = torch.empty(shape, device=x.device, dtype=torch.float32) if out is None else out
        self.set_grad(grads)
        ws = self._reserve(self.train_workspace(B, H, W), x.device)
        with device_of(x):
            check(lib().kdb_model_forward_train(self._h, precision, B, H, W, ptr(x), ptr(sigma), ptr(aug_cond), ptr(class_cond),
                                                ptr(mapping_cond), ptr(cond), self._stride, ptr(u), ptr(out), ptr(grad_x), ptr(ws), ws.numel(),
                                                stream()))
        return out

    def mapping_vjp(self, sigma, dcond, aug_cond=None, class_cond=None, mapping_cond=None, out=None):
        """kdb_model_mapping_vjp: the mapping network's backward for sigma [rows] and dcond [rows, mapping_width] (the gradient of its
        output), conditioning as conditioning() takes it -> (keep [rows, keep floats], grad [rows, grad floats]), their rows laid out as
        mapping_layout gives.  out: a (keep, grad) pair of buffers to write."""
        require_cuda(sigma, dcond, aug_cond, class_cond, mapping_cond)
        c = self.cfg
        rows, L = sigma.numel(), mapping_layout(c.mapping_width, c.mapping_d_ff, c.mapping_depth)
        _fp32_contiguous("model_mapping_vjp", *(t for t in (sigma, dcond, aug_cond, mapping_cond) if t is not None))
        if (tuple(dcond.shape) != (rows, c.mapping_width) or (aug_cond is not None and tuple(aug_cond.shape) != (rows, 9))
                or (mapping_cond is not None and tuple(mapping_cond.shape) != (rows, c.mapping_cond_dim))
                or (class_cond is not None and (class_cond.dtype != torch.int64 or tuple(class_cond.shape) != (rows,)
                                                or not class_cond.is_contiguous()))):
            raise ValueError("model_mapping_vjp: operand shapes do not match")
        keep, grad = (None, None) if out is None else out
        keep = _out(keep, (rows, L["keep"]), dcond, "model_mapping_vjp")
        grad = _out(grad, (rows, L["grad"]), dcond, "model_mapping_vjp")
        require_cuda(keep, grad)
        with device_of(sigma):
            check(lib().kdb_model_mapping_vjp(self._h, rows, ptr(sigma), ptr(aug_cond), ptr(class_cond), ptr(mapping_cond), ptr(dcond), ptr(keep),
                                              ptr(grad), stream()))
        return keep, grad

    def train_forward(self, x, sigma, cond, cond_batch_stride, sigma_data, precision, out=None):
        """kdb_model_train_forward: the forward of forward_train at `precision` (x [B,C,H,W] fp32), bit for bit its `out`."""
        B, _, H, W = x.shape
        if out is None:
            out = torch.empty(B, self.cfg.out_channels, H, W, device=x.device, dtype=torch.float32)
        ws = self._workspace(PREC_FP32, B, H, W, x.device)
        with device_of(x):
            check(lib().kdb_model_train_forward(self._h, precision, B, H, W, ptr(x), ptr(sigma), float(sigma_data), ptr(cond), cond_batch_stride,
                                                ptr(out), ptr(ws), ws.numel(), stream()))
        return out

    def arm_tap(self, name, capacity, device):
        buf = torch.empty(capacity, dtype=torch.float32, device=device)
        check(self._fn("debug_tap")(self._h, name.encode(), ptr(buf), capacity))
        return buf

    def tap_count(self):
        return int(self._fn("tap_count")(self._h))


class UNetEngine(Engine):
    """The image_v1 U-Net at PREC_FP32, PREC_TF32 or PREC_FP16: the Engine calls where the sampler executor makes them, and the parameter
    gradients of training at fp32 (forward_train); no derivative with respect to x."""

    _api = "unet"

    @staticmethod
    def _config(spec):
        cfg = KdbUNetConfig()
        n = len(spec["depths"])
        if n > MAX_LEVELS:
            raise ValueError(f"at most {MAX_LEVELS} levels supported")
        cfg.n_levels, cfg.in_channels, cfg.patch_size, cfg.mapping_out = n, spec["c_in"], spec["patch_size"], spec["feats_in"]
        cfg.mapping_cond_dim, cfg.augment_wrapper = spec["mapping_cond_dim"], int(spec["augment"])
        cfg.skip_stages, cfg.has_variance = spec["skip_stages"], int(spec["has_variance"])
        for i in range(n):
            cfg.depth[i], cfg.channels[i], cfg.self_attn[i] = spec["depths"][i], spec["channels"][i], int(bool(spec["self_attn_depths"][i]))
        return cfg

    def _out_channels(self, x):
        return x.shape[1]

    def conditioning(self, sigma, aug_cond=None, class_cond=None, mapping_cond=None):
        """-> [rows, cond_stride] fp32 table (mapping net + every AdaGN's (weight, bias)); class_cond is refused by the model's front end."""
        require_cuda(sigma, aug_cond, mapping_cond)
        sigma = f32c(sigma)
        rows = sigma.numel()
        aug_cond = None if aug_cond is None else f32c(aug_cond)
        mapping_cond = None if mapping_cond is None else f32c(mapping_cond)
        out = torch.empty(rows, self._stride, device=sigma.device, dtype=torch.float32)
        with device_of(sigma):
            check(lib().kdb_unet_conditioning(self._h, rows, ptr(sigma), ptr(aug_cond), ptr(mapping_cond), ptr(out), stream()))
        return out

    forward_jvp = forward_vjp = unet_has_no_derivative

    def forward_variance(self, x, sigma, cond, cond_batch_stride, sigma_data, precision):
        """kdb_unet_forward_variance: forward()'s output, bit for bit, and the has_variance model's log-variance [B] -> (out, logvar)"""
        B, C, H, W = x.shape
        out = torch.empty_like(x)
        logvar = torch.empty(B, device=x.device, dtype=torch.float32)
        ws = self._workspace(precision, B, H, W, x.device)
        with device_of(x):
            check(lib().kdb_unet_forward_variance(self._h, precision, B, H, W, ptr(x), ptr(sigma), float(sigma_data), ptr(cond), cond_batch_stride,
                                                  ptr(out), ptr(logvar), ptr(ws), ws.numel(), stream()))
        return out, logvar

    def mapping_vjp(self, sigma, dcond, aug_cond=None, mapping_cond=None, out=None):
        """kdb_unet_mapping_vjp: the mapping network's backward for sigma [rows] and dcond [rows, mapping_out] (the gradient of its output)
        -> dict of h0, a0, dz0, dz1, dh0 [rows, mapping_out] and v [rows, mapping_cond_dim].  out: such a dict of buffers to write."""
        require_cuda(sigma, dcond, aug_cond, mapping_cond)
        rows, mw, mcd = sigma.numel(), self.cfg.mapping_out, self.cfg.mapping_cond_dim
        _fp32_contiguous("unet_mapping_vjp", *(t for t in (sigma, dcond, aug_cond, mapping_cond) if t is not None))
        user = mcd - (9 if self.cfg.augment_wrapper else 0)
        if (tuple(dcond.shape) != (rows, mw) or (aug_cond is not None and tuple(aug_cond.shape) != (rows, 9))
                or (mapping_cond is not None and tuple(mapping_cond.shape) != (rows, user))):
            raise ValueError("unet_mapping_vjp: operand shapes do not match")
        out = {} if out is None else out
        res = {k: _out(out.get(k), (rows, mw), dcond, "unet_mapping_vjp") for k in ("h0", "a0", "dz0", "dz1", "dh0")}
        res["v"] = _out(out.get("v"), (rows, mcd), dcond, "unet_mapping_vjp") if mcd else None
        require_cuda(*res.values())
        with device_of(sigma):
            check(lib().kdb_unet_mapping_vjp(self._h, rows, ptr(sigma), ptr(aug_cond), ptr(mapping_cond), ptr(dcond),
                                             *(ptr(res[k]) for k in ("h0", "a0", "dz0", "dz1", "dh0", "v")), stream()))
        return res

    def forward_train(self, x, u, sigma, aug_cond, class_cond, mapping_cond, cond, grads, out=None, grad_x=None, precision=PREC_FP32,
                      dlogvar=None):
        """Parameter gradients at fp32 (kdb_unet_forward_train), with Engine.forward_train's arguments: binds `grads`, then out = F(x) and
        every bound gradient = u^T dF/dparam, plus dlogvar^T dlogvar/dparam when `dlogvar` [B] (the cotangent of a has_variance model's
        log-variance) is given (kdb_unet_forward_train_variance).  The U-Net takes no class_cond and gives no grad_x."""
        if class_cond is not None or grad_x is not None:
            raise ValueError("the image_v1 U-Net takes no class_cond and its training call gives no gradient with respect to x")
        B, C, H, W = x.shape
        if tuple(u.shape) != (B, C, H, W):
            raise ValueError(f"cotangent shape {tuple(u.shape)} != output shape {(B, C, H, W)}")
        if dlogvar is not None and tuple(dlogvar.shape) != (B,):
            raise ValueError(f"dlogvar shape {tuple(dlogvar.shape)} != ({B},)")
        out = torch.empty_like(x) if out is None else out
        self.set_grad(grads)
        ws = self._reserve(self.train_workspace(B, H, W), x.device)
        args = (ptr(x), ptr(sigma), ptr(aug_cond), ptr(mapping_cond), ptr(cond), self._stride, ptr(u))
        with device_of(x):
            if dlogvar is None:
                check(lib().kdb_unet_forward_train(self._h, precision, B, H, W, *args, ptr(out), ptr(ws), ws.numel(), stream()))
            else:
                check(lib().kdb_unet_forward_train_variance(self._h, precision, B, H, W, *args, ptr(f32c(dlogvar)), ptr(out), ptr(ws), ws.numel(),
                                                            stream()))
        return out

    def train_forward(self, x, sigma, cond, cond_batch_stride, sigma_data, precision, out=None):
        """The forward of forward_train: kdb_unet_forward at PREC_FP32 (the U-Net trains at fp32 only), bit for bit its `out`."""
        if precision != PREC_FP32:
            raise NotImplementedError("the image_v1 U-Net trains at fp32 only")
        return self.forward(x, sigma, cond, cond_batch_stride, sigma_data, PREC_FP32, out=out)


class LossRequest(NamedTuple):
    """What `Denoiser.loss` passes, as the keyword `loss_request`, through a DistributedDataParallel wrapper's forward to a native model
    (see `NativeLossCall`), which then returns `request(self.native_loss, x, sigma, **conditioning)`: the training loss runs inside DDP's
    forward, so DDP prepares its reducer, syncs its buffers and honours no_sync() as it does for a torch model.  A NamedTuple, so that
    DDP's input mover carries it through with its tensors on the module's device."""
    kind: int
    noise: torch.Tensor
    sigma_data: float
    weight: object

    def __call__(self, native_loss, input, sigma, **kwargs):
        return native_loss(self.kind, input, self.noise, sigma, self.sigma_data, self.weight, **kwargs)


class NativeLossCall:
    """Base of the modules with a `native_loss` (the native models and KarrasAugmentWrapper): a call with the keyword `loss_request`
    returns that request's native loss instead of running `forward`, whose signature stays the reference's."""

    def __call__(self, *args, loss_request=None, **kwargs):
        if loss_request is None:
            return super().__call__(*args, **kwargs)
        return loss_request(self.native_loss, *args, **kwargs)


class NativeLoss(torch.autograd.Function):
    """A training loss through a native engine with respect to the model's parameters (passed after `keys`, their state-dict names).
    The forward saves the per-element cotangent d loss[b] / d F of the loss kernel (and, for LOSS_VARIANCE, d loss[b] / d logvar[b]); the
    backward scales it by the incoming gradient of each sample's loss and makes one forward_train on the engine `engine()` returns (the
    model's, rebound to its current parameters), which writes every parameter's gradient.  Both run at the model's training precision as the
    forward found it."""

    @staticmethod
    def forward(ctx, model, engine, ev, kind, noise, sigma_data, weight, keys, *params):
        x, sig = ev.x, ev.sigma
        xin = loss_noised_input(x, noise, sig, sigma_data)
        cond = ev.conditioning()
        precision = getattr(model, "train_precision", PREC_FP32)
        dlogvar = None
        if kind == LOSS_VARIANCE:
            f, logvar = ev.engine.forward_variance(xin, sig, cond, ev.engine.cond_stride, 0.0, precision)
            loss, cot, dlogvar = variance_loss(x, noise, sig, sigma_data, f, logvar)
        else:
            w = None if weight is None else f32c(weight).expand(x.shape[0]).contiguous()
            f = ev.engine.train_forward(xin, sig, cond, ev.engine.cond_stride, 0.0, precision)
            loss, cot = denoiser_loss(x, noise, sig, w, sigma_data, f, kind)
        aug, cls, mc = ev.cond
        ctx.model, ctx.engine, ctx.keys, ctx.precision = model, engine, keys, precision
        ctx.save_for_backward(xin, sig, cond, cot, dlogvar, None if aug is None else f32c(aug),
                              None if cls is None else cls.to(torch.int64).contiguous(), None if mc is None else f32c(mc))
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_loss):
        xin, sig, cond, cot, dlogvar, aug, cls, mc = ctx.saved_tensors
        params = dict(ctx.model.named_parameters())
        g = f32c(grad_loss)
        u = cot * g.view(-1, *([1] * (cot.ndim - 1)))
        grads = {k: torch.empty(params[k].shape, device=xin.device, dtype=torch.float32) for k in ctx.keys}
        extra = {} if dlogvar is None else {"dlogvar": dlogvar * g}
        ctx.engine().forward_train(xin, u, sig, aug, cls, mc, cond, grads, precision=ctx.precision, **extra)
        return (None,) * 8 + tuple(grads[k].to(params[k].dtype) for k in ctx.keys)


# ---------------------------------------------------------------------------------------------
# stand-alone kernels (unit tests / profiling)
# ---------------------------------------------------------------------------------------------

@_on_device_of_first
def gemm_bf16(a, w):
    """a [M,K] bf16, w [N,K] bf16 -> [M,N] bf16 on the wgmma kernel (N % 64 == 0, K % 64 == 0)."""
    require_cuda(a, w)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and a.is_contiguous() and w.is_contiguous()
    M, K = a.shape
    N = w.shape[0]
    out = torch.empty(M, N, dtype=torch.bfloat16, device=a.device)
    check(lib().kdb_gemm_bf16(ptr(a), ptr(w), ptr(out), M, N, K, stream()))
    return out


WGRAD_SCRATCH_FLOATS = 1 << 22


def _scratch(t):
    return torch.empty(WGRAD_SCRATCH_FLOATS, device=t.device, dtype=torch.float32)


def _out(out, shape, like, name):
    """out, checked to be a contiguous fp32 tensor of `shape`, or a new one (the entry points write every element)"""
    if out is None:
        return torch.empty(shape, device=like.device, dtype=torch.float32)
    if tuple(out.shape) != tuple(shape) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError(f"{name}: out must be a contiguous fp32 {list(shape)} tensor")
    return out


def _fp32_rows(name, *ts):
    """each a 2-D fp32 tensor with unit column stride (any row stride)"""
    for t in ts:
        if t.dtype != torch.float32 or t.ndim != 2 or t.stride(1) != 1:
            raise ValueError(f"{name}: operands must be 2-D fp32 with contiguous rows, got {t.dtype} {tuple(t.shape)} strides {t.stride()}")


def _fp32_contiguous(name, *ts):
    for t in ts:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"{name}: operands must be contiguous fp32, got {t.dtype} {tuple(t.shape)}")


@_on_device_of_first
def wgrad(dy, x, precision=PREC_FP32, n_rows=None, merge=None, out=None):
    """kdb_wgrad: dW [N, K] = dy[:m]^T x[:m], fp32 (PREC_FP32) or with tf32 operands (truncated) and fp32 accumulation (PREC_TF32).
    dy [m, N] and x [m, K] fp32 with unit column stride (any row stride); merge=(hc, wc): x is instead the fine tokens [B, 2hc, 2wc, Cf] read
    as the TokenMerge gather, K = 4 Cf.  out: an [N, K] fp32 contiguous buffer to write (every element is written)."""
    require_cuda(dy, x, out)
    m = dy.shape[0] if n_rows is None else n_rows
    N = dy.shape[1]
    K = x.shape[-1] * 4 if merge else x.shape[1]
    if dy.dtype != torch.float32 or x.dtype != torch.float32 or dy.ndim != 2 or x.ndim != (4 if merge else 2):
        raise ValueError("wgrad: dy [m, N] and x [m, K] (merge: [B, 2hc, 2wc, Cf]) fp32")
    if dy.stride(1) != 1 or (not merge and x.stride(1) != 1) or (merge and not x.is_contiguous()):
        raise ValueError("wgrad: operands need contiguous rows (the merge gather: contiguous fine tokens)")
    if not 0 < m <= dy.shape[0]:
        raise ValueError(f"wgrad: {m} rows of a dy with {dy.shape[0]}")
    if merge:
        hc, wc = merge
        if hc <= 0 or wc <= 0 or tuple(x.shape[1:3]) != (2 * hc, 2 * wc) or m % (hc * wc) or m // (hc * wc) > x.shape[0]:
            raise ValueError(f"wgrad: fine tokens {tuple(x.shape)} do not hold the TokenMerge gather of {m} rows of a {hc}x{wc} grid")
    elif m > x.shape[0]:
        raise ValueError(f"wgrad: {m} rows of an x with {x.shape[0]}")
    out = _out(out, (N, K), dy, "wgrad")
    hc, wc = merge if merge else (0, 0)
    check(lib().kdb_wgrad(precision, ptr(dy), dy.stride(0), ptr(x), 0 if merge else x.stride(0), ptr(out), m, N, K, hc, wc, ptr(_scratch(dy)),
                          stream()))
    return out



def wgrad_tf32(dy, x, n_rows=None, merge=None, out=None):
    """wgrad at PREC_TF32: the tf32 training precision's weight gradient (kdb_wgrad with tf32 operands), same arguments"""
    return wgrad(dy, x, PREC_TF32, n_rows=n_rows, merge=merge, out=out)


@_on_device_of_first
def wgrad_patch_in(dtok, x, patch, out=None):
    """kdb_wgrad_patch_in: dW [N, ph pw C] = dtok^T P with P the patch rows (columns (ph pw c)) of the NCHW image x [B, C, H, W] and
    dtok [B (H/ph) (W/pw), N] contiguous fp32"""
    require_cuda(dtok, x, out)
    _fp32_contiguous("wgrad_patch_in", dtok, x)
    (ph, pw), (B, C, H, W) = patch, x.shape
    if ph <= 0 or pw <= 0 or H % ph or W % pw or dtok.ndim != 2 or dtok.shape[0] != B * (H // ph) * (W // pw):
        raise ValueError(f"wgrad_patch_in: dtok {tuple(dtok.shape)} is not one row per {ph}x{pw} patch of an image {tuple(x.shape)}")
    N = dtok.shape[1]
    out = _out(out, (N, ph * pw * C), dtok, "wgrad_patch_in")
    check(lib().kdb_wgrad_patch_in(ptr(dtok), ptr(x), ptr(out), B, C, H, W, ph, pw, N, ptr(_scratch(x)), stream()))
    return out


@_on_device_of_first
def wgrad_patch_out(u, tokens, scale, rstd, patch, out=None):
    """kdb_wgrad_patch_out: dW [ph pw C, C0] = P^T (tokens * (scale * rstd)) with P the patch rows (columns (ph pw c)) of u [B, C, H, W],
    tokens [B (H/ph) (W/pw), C0], scale [C0] and rstd [B (H/ph) (W/pw)], all contiguous fp32"""
    require_cuda(u, tokens, scale, rstd, out)
    _fp32_contiguous("wgrad_patch_out", u, tokens, scale, rstd)
    (ph, pw), (B, C, H, W) = patch, u.shape
    T = B * (H // ph) * (W // pw) if ph > 0 and pw > 0 else -1
    if ph <= 0 or pw <= 0 or H % ph or W % pw or tokens.ndim != 2 or tokens.shape[0] != T or tuple(rstd.shape) != (T,) or \
            tuple(scale.shape) != (tokens.shape[1],):
        raise ValueError(f"wgrad_patch_out: tokens {tuple(tokens.shape)}, scale {tuple(scale.shape)} and rstd {tuple(rstd.shape)} do not match "
                         f"{ph}x{pw} patches of {tuple(u.shape)}")
    C0 = tokens.shape[1]
    out = _out(out, (ph * pw * C, C0), u, "wgrad_patch_out")
    check(lib().kdb_wgrad_patch_out(ptr(u), ptr(tokens), ptr(scale), ptr(rstd), ptr(out), B, C, H, W, ph, pw, C0, ptr(_scratch(u)), stream()))
    return out


@_on_device_of_first
def norm_scale_grad(x, dy, rows_per_image=None, out=None, ldo=None):
    """kdb_norm_scale_grad: the RMSNorm scale gradient per image, sum over each image's rows of dy * x * rsqrt(mean(x^2) + 1e-6); x and dy
    [rows, C] fp32 with contiguous rows (any row stride), rows_per_image (default: all rows, one image).  -> [B, C], or written into out
    (flat, contiguous) at out[b * ldo + c] (ldo default C)"""
    require_cuda(x, dy, out)
    _fp32_rows("norm_scale_grad", x, dy)
    rows, C = x.shape
    R = rows if rows_per_image is None else rows_per_image
    if tuple(dy.shape) != (rows, C) or R <= 0 or rows % R:
        raise ValueError(f"norm_scale_grad: x {tuple(x.shape)}, dy {tuple(dy.shape)} with {R} rows per image")
    B, ldo = rows // R, C if ldo is None else ldo
    if out is None:
        out = torch.empty(B, C, device=x.device, dtype=torch.float32)
        ldo = C
    elif out.dtype != torch.float32 or not out.is_contiguous() or (B > 1 and ldo < C) or out.numel() < (B - 1) * ldo + C:
        raise ValueError(f"norm_scale_grad: out {tuple(out.shape)} does not hold {B} images of {C} channels {ldo} apart")
    check(lib().kdb_norm_scale_grad(ptr(x), x.stride(0), ptr(dy), dy.stride(0), ptr(out), ldo, R, rows, C, ptr(_scratch(x)), stream()))
    return out


@_on_device_of_first
def colsum(p, out=None):
    """kdb_colsum: the column sums [C] of p [rows, C] contiguous fp32"""
    require_cuda(p, out)
    _fp32_contiguous("colsum", p)
    if p.ndim != 2:
        raise ValueError(f"colsum: p must be [rows, C], got {tuple(p.shape)}")
    out = _out(out, (p.shape[1],), p, "colsum")
    check(lib().kdb_colsum(ptr(p), p.shape[0], p.shape[1], ptr(out), ptr(_scratch(p)), stream()))
    return out


@_on_device_of_first
def split_fac_grad(y, skip, dup, out=None):
    """kdb_split_fac_grad: TokenSplit's fac gradient [1], the sum of (y - skip) dup with y [B, H/2, W/2, 4C] in TokenMerge order and skip,
    dup [B, H, W, C], all contiguous fp32"""
    require_cuda(y, skip, dup, out)
    _fp32_contiguous("split_fac_grad", y, skip, dup)
    B, H, W, C = skip.shape
    if tuple(dup.shape) != (B, H, W, C) or H % 2 or W % 2 or tuple(y.shape) != (B, H // 2, W // 2, 4 * C):
        raise ValueError(f"split_fac_grad: y {tuple(y.shape)}, skip {tuple(skip.shape)}, dup {tuple(dup.shape)}")
    out = _out(out, (1,), y, "split_fac_grad")
    check(lib().kdb_split_fac_grad(ptr(y), ptr(skip), ptr(dup), ptr(out), B, H, W, C, ptr(_scratch(y)), stream()))
    return out


@_on_device_of_first
def class_emb_grad(demb, cls, n_classes, out=None):
    """kdb_class_emb_grad: [n_classes, mw], row j the sum of the rows of demb [rows, mw] (fp32, contiguous rows) whose class cls [rows]
    (int64) is j"""
    require_cuda(demb, cls, out)
    _fp32_rows("class_emb_grad", demb)
    rows, mw = demb.shape
    if cls.dtype != torch.int64 or tuple(cls.shape) != (rows,) or not cls.is_contiguous():
        raise ValueError(f"class_emb_grad: cls must be contiguous int64 [{rows}], got {cls.dtype} {tuple(cls.shape)}")
    out = _out(out, (n_classes, mw), demb, "class_emb_grad")
    check(lib().kdb_class_emb_grad(ptr(demb), demb.stride(0), ptr(cls), ptr(out), rows, n_classes, mw, stream()))
    return out


VJP_STORE, VJP_UNPATCH_ACC = 0, 1


def _shaped(name, t, shape):
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name}: {tuple(t.shape)} where {list(shape)} is needed")


@_on_device_of_first
def gemm_vjp(dc, w, out=None, unpatch=None):
    """kdb_gemm_vjp: the input gradient dA [M, K] = dc [M, N] w [N, K] of a Linear, contiguous fp32 (N, K multiples of 4).  unpatch=(hc, wc):
    the rows are coarse tokens of hc x wc grids and dA is ADDED to out, the fine tokens [M / (hc wc), 2 hc, 2 wc, K / 4] (required), through
    the TokenMerge un-patch."""
    require_cuda(dc, w, out)
    _fp32_contiguous("gemm_vjp", dc, w)
    if dc.ndim != 2 or w.ndim != 2 or dc.shape[1] != w.shape[0]:
        raise ValueError(f"gemm_vjp: dc {tuple(dc.shape)} and w {tuple(w.shape)} do not chain")
    (M, N), K = dc.shape, w.shape[1]
    hc, wc = unpatch or (0, 0)
    if unpatch:
        if out is None or hc <= 0 or wc <= 0 or K % 4 or M % (hc * wc):
            raise ValueError(f"gemm_vjp: {M} x {K} does not un-patch onto {hc}x{wc} coarse grids, or no fine tokens to add to")
        _fp32_contiguous("gemm_vjp", out)
        _shaped("gemm_vjp", out, (M // (hc * wc), 2 * hc, 2 * wc, K // 4))
    else:
        out = _out(out, (M, K), dc, "gemm_vjp")
    check(lib().kdb_gemm_vjp(ptr(dc), ptr(w), ptr(out), M, N, K, VJP_UNPATCH_ACC if unpatch else VJP_STORE, hc, wc, K // 4 if unpatch else 0,
                             stream()))
    return out


@_on_device_of_first
def rmsnorm_vjp(x, dy, scale, out, rows_per_image=None, scale_bstride=0):
    """kdb_rmsnorm_vjp: ADDS the input gradient of an (Ada)RMSNorm to out (returned), x, dy and out [rows, C] contiguous fp32; the scale row
    of image b (rows_per_image rows each, default all) starts at scale[b * scale_bstride] (0: one row shared by all)"""
    require_cuda(x, dy, scale, out)
    _fp32_contiguous("rmsnorm_vjp", x, dy, scale, out)
    rows, C = x.shape
    R = rows if rows_per_image is None else rows_per_image
    _shaped("rmsnorm_vjp", dy, (rows, C))
    _shaped("rmsnorm_vjp", out, (rows, C))
    if R <= 0 or rows % R or scale_bstride < 0 or scale.numel() < (rows // R - 1) * scale_bstride + C:
        raise ValueError(f"rmsnorm_vjp: {rows} rows of {R} per image, or a scale of {scale.numel()} floats for rows {scale_bstride} apart")
    check(lib().kdb_rmsnorm_vjp(ptr(x), ptr(dy), ptr(out), ptr(scale), scale_bstride, R, rows, C, stream()))
    return out


@_on_device_of_first
def qknorm_rope_vjp(qkv, dqkv, pos, freqs, scale, eps, r, dscale_rows=None):
    """kdb_qknorm_rope_vjp: in place on the q and k thirds of dqkv [rows, 3, nh, e] (returned with dscale_rows), qkv the primal before the
    cosine-sim scale and RoPE, pos [T, 2] (rows a multiple of T), freqs [nh, r / 2], scale [nh]; dscale_rows: None or an [rows, nh] buffer
    for each (row, head)'s term of the head scale's gradient.  All contiguous fp32."""
    require_cuda(qkv, dqkv, pos, freqs, scale, dscale_rows)
    _fp32_contiguous("qknorm_rope_vjp", *(t for t in (qkv, dqkv, pos, freqs, scale, dscale_rows) if t is not None))
    if qkv.ndim != 4 or qkv.shape[1] != 3 or pos.ndim != 2 or pos.shape[1] != 2:
        raise ValueError(f"qknorm_rope_vjp: qkv {tuple(qkv.shape)} is no [rows, 3, nh, e], or pos {tuple(pos.shape)} no [T, 2]")
    rows, _, nh, e = qkv.shape
    T = pos.shape[0]
    _shaped("qknorm_rope_vjp", dqkv, qkv.shape)
    _shaped("qknorm_rope_vjp", freqs, (nh, r // 2))
    _shaped("qknorm_rope_vjp", scale, (nh,))
    if dscale_rows is not None:
        _shaped("qknorm_rope_vjp", dscale_rows, (rows, nh))
    if T <= 0 or rows % T:
        raise ValueError(f"qknorm_rope_vjp: {rows} rows are no whole images of {T} tokens")
    check(lib().kdb_qknorm_rope_vjp(ptr(qkv), ptr(dqkv), ptr(pos), ptr(freqs), ptr(scale), float(eps), r, rows, T, nh, e, ptr(dscale_rows),
                                    stream()))
    return dqkv, dscale_rows


@_on_device_of_first
def geglu_vjp(h, dy, out=None):
    """kdb_geglu_vjp: h [M, 2F] (value | gate), dy [M, F] contiguous fp32 -> dh [M, 2F]"""
    require_cuda(h, dy, out)
    _fp32_contiguous("geglu_vjp", h, dy)
    M, F = dy.shape
    _shaped("geglu_vjp", h, (M, 2 * F))
    out = _out(out, (M, 2 * F), h, "geglu_vjp")
    check(lib().kdb_geglu_vjp(ptr(h), ptr(dy), ptr(out), M, F, stream()))
    return out


def _fine_and_coarse(name, fine, coarse, fac=None):
    """fine [B, H, W, C] and coarse [B, H/2, W/2, 4C] contiguous fp32 (fac: one fp32 float) -> (B, H, W, C)"""
    _fp32_contiguous(name, fine, coarse, *(() if fac is None else (fac,)))
    if fine.ndim != 4 or fine.shape[1] % 2 or fine.shape[2] % 2 or (fac is not None and fac.numel() != 1):
        raise ValueError(f"{name}: {tuple(fine.shape)} is no [B, H, W, C] with H and W even, or fac is not one float")
    B, H, W, C = fine.shape
    _shaped(name, coarse, (B, H // 2, W // 2, 4 * C))
    return B, H, W, C


@_on_device_of_first
def split_vjp_gather(dup, fac, out=None):
    """kdb_split_vjp_gather: TokenSplit's lerp backward, dup [B, H, W, C] -> out [B, H/2, W/2, 4C] = fac dup in TokenMerge order, and
    dup *= 1 - fac IN PLACE; fac one fp32 float on the device"""
    require_cuda(dup, fac, out)
    B, H, W, C = dup.shape
    out = _out(out, (B, H // 2, W // 2, 4 * C), dup, "split_vjp_gather")
    _fine_and_coarse("split_vjp_gather", dup, out, fac)
    check(lib().kdb_split_vjp_gather(ptr(dup), ptr(out), ptr(fac), B, H, W, C, stream()))
    return out


@_on_device_of_first
def split_unpatch_lerp(y, skip, fac, out=None):
    """kdb_split_unpatch_lerp: torch.lerp(skip, unpatch2x2(y), fac) -> [B, H, W, C], y [B, H/2, W/2, 4C], skip [B, H, W, C], fac one float"""
    require_cuda(y, skip, fac, out)
    B, H, W, C = _fine_and_coarse("split_unpatch_lerp", skip, y, fac)
    out = _out(out, skip.shape, skip, "split_unpatch_lerp")
    check(lib().kdb_split_unpatch_lerp(ptr(y), ptr(skip), ptr(fac), ptr(out), B, H, W, C, stream()))
    return out


@_on_device_of_first
def merge_scatter_add(d, out):
    """kdb_merge_scatter_add: out [B, H, W, C] += unpatch2x2(d), d [B, H/2, W/2, 4C]; returns out"""
    require_cuda(d, out)
    B, H, W, C = _fine_and_coarse("merge_scatter_add", out, d)
    check(lib().kdb_merge_scatter_add(ptr(d), ptr(out), B, H, W, C, stream()))
    return out


def _patch_grid(name, size, patch, sigma, sigma_data):
    (B, C, H, W), (ph, pw) = size, patch
    if ph <= 0 or pw <= 0 or H % ph or W % pw:
        raise ValueError(f"{name}: a {H}x{W} image in {ph}x{pw} patches")
    if sigma_data > 0:
        if sigma is None:
            raise ValueError(f"{name}: sigma_data > 0 needs sigma")
        _fp32_contiguous(name, sigma)
        _shaped(name, sigma, (B,))
    return B * (H // ph) * (W // pw)


@_on_device_of_first
def patch_out_vjp(tokens, norm_scale, w, u, patch, sigma=None, sigma_data=0.0, out=None, dnorm=None, rstd=None):
    """kdb_patch_out_vjp: out_norm + patch_out's backward, tokens [T, C0], norm_scale [C0], w [ph pw C, C0], u [B, C, H, W] the output's
    gradient (scaled by Karras's c_out of sigma [B] when sigma_data > 0) -> (dtokens [T, C0], dnorm, rstd): dnorm [T, C0] and rstd [T] are
    written where given.  All contiguous fp32."""
    require_cuda(tokens, norm_scale, w, u, sigma, out, dnorm, rstd)
    _fp32_contiguous("patch_out_vjp", tokens, norm_scale, w, u, *(t for t in (dnorm, rstd) if t is not None))
    T = _patch_grid("patch_out_vjp", u.shape, patch, sigma, sigma_data)
    C0 = tokens.shape[-1]
    _shaped("patch_out_vjp", tokens, (T, C0))
    _shaped("patch_out_vjp", norm_scale, (C0,))
    _shaped("patch_out_vjp", w, (patch[0] * patch[1] * u.shape[1], C0))
    if dnorm is not None:
        _shaped("patch_out_vjp", dnorm, (T, C0))
    if rstd is not None:
        _shaped("patch_out_vjp", rstd, (T,))
    out = _out(out, (T, C0), tokens, "patch_out_vjp")
    (B, C, H, W), (ph, pw) = u.shape, patch
    check(lib().kdb_patch_out_vjp(ptr(tokens), ptr(norm_scale), ptr(w), ptr(u), ptr(sigma), float(sigma_data), ptr(out), B, C, H, W, ph, pw, C0,
                                  ptr(dnorm), ptr(rstd), stream()))
    return out, dnorm, rstd


@_on_device_of_first
def patch_in_vjp(dtokens, w, size, patch, u=None, sigma=None, sigma_data=0.0, out=None):
    """kdb_patch_in_vjp: patch_in's backward to an image of size (B, C, H, W): unpatch(dtokens [T, N] w [N, ph pw C]), with sigma_data > 0
    c_skip u + c_in unpatch(...) (u [B, C, H, W] the output's gradient, sigma [B]).  All contiguous fp32."""
    require_cuda(dtokens, w, u, sigma, out)
    _fp32_contiguous("patch_in_vjp", dtokens, w, *(() if u is None else (u,)))
    T = _patch_grid("patch_in_vjp", size, patch, sigma, sigma_data)
    N = dtokens.shape[-1]
    _shaped("patch_in_vjp", dtokens, (T, N))
    _shaped("patch_in_vjp", w, (N, patch[0] * patch[1] * size[1]))
    if sigma_data > 0:
        if u is None:
            raise ValueError("patch_in_vjp: sigma_data > 0 needs u")
        _shaped("patch_in_vjp", u, size)
    out = _out(out, tuple(size), dtokens, "patch_in_vjp")
    (B, C, H, W), (ph, pw) = size, patch
    check(lib().kdb_patch_in_vjp(ptr(dtokens), ptr(w), ptr(u), ptr(sigma), float(sigma_data), ptr(out), B, C, H, W, ph, pw, N, stream()))
    return out


def mapping_layout(mw, dff, depth):
    """The row layout of kdb_model_mapping_vjp's keep and grad (the header's formulas): their widths and each vector's offset"""
    f4 = (dff + 3) // 4 * 4
    blk = mw + 2 * dff + f4
    xn = lambda l: (4 + depth) * mw + l * blk
    dxn = lambda l: (depth + 1) * mw + l * (mw + 2 * dff)
    return {"keep": xn(depth), "grad": dxn(depth) + mw, "ff_t": 0, "ff_a": mw, "emb": 2 * mw, "r": lambda l: (3 + l) * mw, "xn": xn,
            "up": lambda l: xn(l) + mw, "g": lambda l: xn(l) + mw + 2 * dff, "dr": lambda l: l * mw, "dxn": dxn,
            "dh": lambda l: dxn(l) + mw, "demb": dxn(depth)}


def interleave_geglu_rows(w_up):
    """up_proj.weight [2F, K] -> the value/gate row interleave the fused GEGLU epilogue expects (8 value rows, 8 gate rows)."""
    F2, K = w_up.shape
    F = F2 // 2
    val, gate = w_up[:F].reshape(F // 8, 8, K), w_up[F:].reshape(F // 8, 8, K)
    return torch.cat([val, gate], dim=1).reshape(F2, K).contiguous()


@_on_device_of_first
def gemm_bf16_geglu(a, w_up, ss_in=None):
    """a [M,K] bf16, w_up [2F,K] bf16 (reference row order) -> value * gelu(gate) [M,F] bf16 on the wgmma kernel."""
    require_cuda(a, w_up, ss_in)
    assert a.dtype == torch.bfloat16 and w_up.dtype == torch.bfloat16 and a.is_contiguous()
    M, K = a.shape
    N2 = w_up.shape[0]
    w_il = interleave_geglu_rows(w_up)
    out = torch.empty(M, N2 // 2, dtype=torch.bfloat16, device=a.device)
    check(lib().kdb_gemm_bf16_geglu(ptr(a), ptr(w_il), ptr(out), M, N2, K, ptr(ss_in), stream()))
    return out


@_on_device_of_first
def ffn_fused_bf16(x, w_up, w_down, ss_in, ss_out=None):
    """x [M,128] bf16 (updated IN PLACE and returned), w_up [2F,128] bf16 (reference row order), w_down [128,F] bf16, ss_in [M,8] fp32 with
    sum(x^2) per row in slot 0: x <- x + (value * gelu(gate))(x / rms(x)) @ w_down^T in one kernel (tc_ffn_fused.cuh)."""
    require_cuda(x, w_up, w_down, ss_in, ss_out)
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and w_down.is_contiguous() and ss_in.dtype == torch.float32
    M, F = x.shape[0], w_down.shape[1]
    w_il = interleave_geglu_rows(w_up)
    check(lib().kdb_ffn_fused_bf16(ptr(x), ptr(w_il), ptr(w_down), M, F, ptr(ss_in), ptr(ss_out), stream()))
    return x


@_on_device_of_first
def attn_block_bf16(x, w_qkv, w_out, theta, scale, shift, ss_in, ss_out):
    """x [B,h,w,128] bf16 (updated IN PLACE and returned), w_qkv [384,128] and w_out [128,128] bf16, theta [h,w,2,16] fp32 RoPE angles as
    the reference's AxialRoPE makes them (pos * freqs, y then x), scale [2] fp32, shift 0 or 4, ss_in / ss_out [B*h*w,8] fp32 (sum(x^2)
    per row in slot 0): x <- x + out_proj(shifted_window_attn(qkv(x / rms(x)))) in one kernel (tc_attn_block.cuh)."""
    require_cuda(x, w_qkv, w_out, theta, scale, ss_in, ss_out)
    assert x.dtype == torch.bfloat16 and x.is_contiguous() and w_qkv.is_contiguous() and w_out.is_contiguous()
    assert ss_in.dtype == torch.float32 and ss_out.dtype == torch.float32 and scale.dtype == torch.float32
    B, h, w, _ = x.shape
    # [h,w,2,16] -> [2][8][h*w] x (cos t_2i, cos t_2i+1, sin t_2i, sin t_2i+1)
    th = theta.float().reshape(h * w, 2, 8, 2).permute(1, 2, 0, 3)
    table = torch.cat([th.cos(), th.sin()], dim=-1).contiguous()
    check(lib().kdb_attn_block_bf16(ptr(x), ptr(w_qkv), ptr(w_out), ptr(table), ptr(scale.contiguous()), B, h, w, shift, ptr(ss_in), ptr(ss_out),
                                    stream()))
    return x


@_on_device_of_first
def attention(qkv, h, w, n_heads, d_head, attn_type, attn_param=0, shift=0, fast=False, logit_bound=None):
    """qkv [B, h*w, 3*n_heads*d_head] (fp32 or bf16, q/k already normalised + rotated) -> [B, h*w, n_heads*d_head].
    logit_bound: optional fp32 [n_heads] with |q . k| <= bound (the cosine-similarity scale): single-pass fixed-shift softmax."""
    require_cuda(qkv, logit_bound)
    prec = PREC_BF16 if qkv.dtype == torch.bfloat16 else PREC_FP32
    B = qkv.shape[0]
    out = torch.empty(B, h * w, n_heads * d_head, dtype=qkv.dtype, device=qkv.device)
    code = _ATTN_CODE[attn_type] if isinstance(attn_type, str) else attn_type
    check(lib().kdb_attention(prec, 1 if fast else 0, ptr(qkv.contiguous()), ptr(out), B, h, w, n_heads, d_head, code, attn_param, shift,
                               ptr(logit_bound), stream()))
    return out


def _unet_conv(fn, x1, w, ksize, x2, bias, r1, r2, out, w_dtype=torch.float32):
    require_cuda(x1, w, x2, bias, r1, r2, out)
    B, h, wd, c1 = x1.shape
    N = w.shape[0]
    c2 = 0 if x2 is None else x2.shape[-1]
    rc1 = 0 if r1 is None else r1.shape[-1]
    if out is None:
        out = torch.empty(B, h, wd, N, dtype=torch.float32, device=x1.device)
    x1, x2, bias, r1, r2 = (None if t is None else f32c(t) for t in (x1, x2, bias, r1, r2))
    w = w.to(w_dtype).contiguous()
    check(fn(ptr(x1), c1, ptr(x2), c2, ptr(w), ptr(bias), ptr(r1), rc1, ptr(r2), ptr(out), B, h, wd, N, ksize, stream()))
    return out


@_on_device_of_first
def unet_conv(x1, w, ksize, x2=None, bias=None, r1=None, r2=None, out=None):
    """The U-Net engine's convolution (kdb_unet_conv): x1 [B,h,w,c1] and x2 [B,h,w,c2] token-major fp32 (their channel concatenation is
    the input), w the tap-major weight [N, ksize*ksize, c1 + c2], bias [N], the residual [B,h,w,N] given as r1 (the first rc1 channels,
    all N without r2) and r2 (the rest) -> out [B,h,w,N]."""
    return _unet_conv(lib().kdb_unet_conv, x1, w, ksize, x2, bias, r1, r2, out)


@_on_device_of_first
def unet_conv_tf32(x1, w, ksize, x2=None, bias=None, r1=None, r2=None, out=None):
    """unet_conv on the tensor cores (kdb_unet_conv_tf32): the same arguments; the products take the inputs and w truncated to tf32 (round
    w to tf32 first for round-to-nearest weights, as the engine does) and accumulate in fp32."""
    return _unet_conv(lib().kdb_unet_conv_tf32, x1, w, ksize, x2, bias, r1, r2, out)


@_on_device_of_first
def unet_conv_fp16(x1, w, ksize, x2=None, bias=None, r1=None, r2=None, out=None):
    """unet_conv with fp16 operands (kdb_unet_conv_fp16): the same arguments; w (fp32 or fp16, tap-major [N, ksize*ksize, c1 + c2]) is
    rounded to fp16 (nearest even, as the engine's finalize does) and padded to the kernel's row length, the inputs are rounded to fp16 in
    the kernel; fp32 accumulation.  Rounding does not saturate: an operand of magnitude >= 65520 becomes inf."""
    require_cuda(w)
    ct = w.shape[-1]
    w16 = torch.zeros(*w.shape[:-1], (ct + 7) // 8 * 8, dtype=torch.float16, device=w.device)
    w16[..., :ct] = w
    return _unet_conv(lib().kdb_unet_conv_fp16, x1, w16, ksize, x2, bias, r1, r2, out, w_dtype=torch.float16)


@_on_device_of_first
def unet_conv_wgrad(dy, x1, ksize, x2=None, out=None):
    """kdb_unet_conv_wgrad: the weight gradient [N, c1 + c2, ksize, ksize] of unet_conv, dy [B, h, w, N] and x1, x2 [B, h, w, c] token-major
    fp32 contiguous"""
    require_cuda(dy, x1, x2, out)
    _fp32_contiguous("unet_conv_wgrad", *(t for t in (dy, x1, x2) if t is not None))
    B, h, w, N = dy.shape
    c2 = 0 if x2 is None else x2.shape[-1]
    if x1.shape[:3] != dy.shape[:3] or (x2 is not None and x2.shape[:3] != dy.shape[:3]):
        raise ValueError("unet_conv_wgrad: dy and the inputs must share [B, h, w]")
    out = _out(out, (N, x1.shape[-1] + c2, ksize, ksize), dy, "unet_conv_wgrad")
    check(lib().kdb_unet_conv_wgrad(ptr(dy), N, ptr(x1), x1.shape[-1], ptr(x2), c2, ptr(out), B, h, w, ksize, ptr(_scratch(dy)), stream()))
    return out


@_on_device_of_first
def unet_adagn_vjp(x1, dy, cond, ada_off, groups, gelu, x2=None, add=None, dss=None, out=None):
    """kdb_unet_adagn_vjp: x1 [B, h, w, c1] (and x2 [B, h, w, c2]) the AdaGN input, dy the gradient of its output, cond [B, stride] rows ->
    (dx1, dx2 or None, dss [B, stride]: the mapper-output gradients at ada_off, the rest as passed in or NaN).  out: (dx1, dx2 or None)
    buffers to write, of x1's and x2's shapes."""
    require_cuda(x1, dy, cond, x2, add, dss)
    _fp32_contiguous("unet_adagn_vjp", *(t for t in (x1, dy, cond, x2, add, dss) if t is not None))
    B, h, w, c1 = x1.shape
    c2 = 0 if x2 is None else x2.shape[-1]
    if tuple(dy.shape) != (B, h, w, c1 + c2) or (add is not None and add.shape != dy.shape) or cond.shape[0] != B:
        raise ValueError("unet_adagn_vjp: operand shapes do not match")
    if ada_off < 0 or any(t is not None and (t.shape[0] != B or ada_off + 2 * (c1 + c2) > t.shape[1]) for t in (cond, dss)):
        raise ValueError("unet_adagn_vjp: the (weight, bias) pair lies outside the conditioning row")
    o1, o2 = (None, None) if out is None else out
    dx1 = _out(o1, x1.shape, x1, "unet_adagn_vjp")
    dx2 = None if x2 is None else _out(o2, x2.shape, x2, "unet_adagn_vjp")
    require_cuda(dx1, dx2)
    dss = torch.full_like(cond, float("nan")) if dss is None else dss
    check(lib().kdb_unet_adagn_vjp(ptr(x1), c1, ptr(x2), c2, ptr(dy), ptr(add), ptr(dx1), ptr(dx2), ptr(cond), cond.shape[1], ada_off, ptr(dss),
                                   dss.shape[1], groups, int(gelu), B, h * w, stream()))
    return dx1, dx2, dss


@_on_device_of_first
def unet_flip_conv_weight(w):
    """kdb_unet_flip_conv_weight: tap-major w [N, ksize^2, C] fp32 -> the input-gradient convolution's weight [C, ksize^2, N]"""
    require_cuda(w)
    _fp32_contiguous("unet_flip_conv_weight", w)
    N, kk, C = w.shape
    if kk not in (1, 9):
        raise ValueError(f"unet_flip_conv_weight: {kk} taps")
    out = torch.empty(C, kk, N, device=w.device, dtype=torch.float32)
    check(lib().kdb_unet_flip_conv_weight(ptr(w), ptr(out), N, C, 1 if kk == 1 else 3, stream()))
    return out


@_on_device_of_first
def unet_resample_vjp(dout, h, w, up, add=None, out=None):
    """kdb_unet_resample_vjp: the adjoint of the 2x down- (up = False) or upsampling of an h x w grid, dout [B, h', w', C] -> [B, h, w, C]
    (+ add, which may be out itself)"""
    require_cuda(dout, add, out)
    _fp32_contiguous("unet_resample_vjp", *(t for t in (dout, add) if t is not None))
    B, ho, wo, C = dout.shape
    if (ho, wo) != ((2 * h, 2 * w) if up else (h // 2, w // 2)):
        raise ValueError(f"unet_resample_vjp: a {ho}x{wo} gradient is not the output grid of a {h}x{w} input")
    din = _out(out, (B, h, w, C), dout, "unet_resample_vjp")
    if add is not None and tuple(add.shape) != tuple(din.shape):
        raise ValueError("unet_resample_vjp: add must have the input's shape")
    check(lib().kdb_unet_resample_vjp(ptr(dout), ptr(add), ptr(din), B, h, w, C, int(up), stream()))
    return din


@_on_device_of_first
def unet_proj_out_vjp(u, w, out=None):
    """kdb_unet_proj_out_vjp: proj_out's input gradient u [M, N] @ w [N, K] -> [M, K], u and w contiguous fp32"""
    require_cuda(u, w, out)
    _fp32_contiguous("unet_proj_out_vjp", u, w)
    (M, N), K = u.shape, w.shape[-1]
    if w.ndim != 2 or w.shape[0] != N:
        raise ValueError(f"unet_proj_out_vjp: u {tuple(u.shape)} and w {tuple(w.shape)} do not chain")
    out = _out(out, (M, K), u, "unet_proj_out_vjp")
    check(lib().kdb_unet_proj_out_vjp(ptr(u), ptr(w), ptr(out), M, N, K, stream()))
    return out


@_on_device_of_first
def unet_unshuffle(x, p, ld=None, out=None):
    """kdb_unet_unshuffle: pixel_unshuffle of an NCHW x [B, C, H, W] fp32 -> token rows [B (H/p) (W/p), ld], column (c, i, j);
    ld defaults to C p p, columns past it are zero"""
    require_cuda(x, out)
    _fp32_contiguous("unet_unshuffle", x)
    B, C, H, W = x.shape
    ld = C * p * p if ld is None else ld
    if p < 1 or H % p or W % p or ld < C * p * p:
        raise ValueError(f"unet_unshuffle: {H}x{W} by {p} into rows of {ld}")
    out = _out(out, (B * (H // p) * (W // p), ld), x, "unet_unshuffle")
    check(lib().kdb_unet_unshuffle(ptr(x), ptr(out), B, C, H, W, p, ld, stream()))
    return out


def _unet_attention(precision, qkv, h, w, n_heads, d_head):
    require_cuda(qkv)
    B = qkv.shape[0]
    out = torch.empty(B, h * w, n_heads * d_head, dtype=torch.float32, device=qkv.device)
    check(lib().kdb_attention(precision, 0, ptr(f32c(qkv)), ptr(out), B, h, w, n_heads, d_head, ATTN_GLOBAL, 0, 0, None, stream()))
    return out


@_on_device_of_first
def unet_attention_tf32(qkv, h, w, n_heads, d_head=64):
    """The U-Net engine's global attention at tf32 (kdb_attention with PREC_TF32): qkv [B, h*w, 3*n_heads*d_head] fp32 in (t nh e) order,
    1/sqrt(d_head) already in q -> [B, h*w, n_heads*d_head] fp32.  q, k, v and the probabilities are truncated to tf32; d_head 64."""
    return _unet_attention(PREC_TF32, qkv, h, w, n_heads, d_head)


@_on_device_of_first
def unet_attention_fp16(qkv, h, w, n_heads, d_head=64):
    """unet_attention_tf32 at fp16 (kdb_attention with PREC_FP16): q, k, v and the probabilities are rounded to fp16 (nearest even); the
    scores, the softmax and its sum stay fp32."""
    return _unet_attention(PREC_FP16, qkv, h, w, n_heads, d_head)


def _fp32_attention_args(tensors, numels):
    for t, n in zip(tensors, numels):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n:
            raise ValueError(f"the attention derivatives take contiguous fp32 tensors of the attention's shape (got {t.dtype} {tuple(t.shape)})")


@_on_device_of_first
def attention_jvp(qkv, dqkv, h, w, n_heads, d_head, attn_type, attn_param=0, shift=0, out=None):
    """Tangent of the fp32 attention(qkv) along dqkv (both [B, h*w, 3*n_heads*d_head]) -> [B, h*w, n_heads*d_head]."""
    require_cuda(qkv, dqkv, out)
    B = qkv.shape[0]
    out = torch.empty(B, h * w, n_heads * d_head, dtype=torch.float32, device=qkv.device) if out is None else out
    T = B * h * w * n_heads * d_head
    _fp32_attention_args((qkv, dqkv, out), (3 * T, 3 * T, T))
    code = _ATTN_CODE[attn_type] if isinstance(attn_type, str) else attn_type
    check(lib().kdb_attention_jvp(ptr(qkv), ptr(dqkv), ptr(out), B, h, w, n_heads, d_head, code, attn_param, shift, stream()))
    return out


@_on_device_of_first
def attention_vjp(qkv, out, dout, h, w, n_heads, d_head, attn_type, attn_param=0, shift=0, dqkv=None, stats=None):
    """Gradient of the fp32 attention(qkv) for the output gradient dout: qkv [B, h*w, 3*n_heads*d_head], out = attention(qkv) and dout
    [B, h*w, n_heads*d_head] -> dqkv like qkv.  stats: optional scratch [B, n_heads, h*w, 3] fp32 (the per-query softmax statistics)."""
    require_cuda(qkv, out, dout, dqkv, stats)
    B = qkv.shape[0]
    dqkv = torch.empty_like(qkv) if dqkv is None else dqkv
    stats = torch.empty(B, n_heads, h * w, 3, dtype=torch.float32, device=qkv.device) if stats is None else stats
    T = B * h * w * n_heads * d_head
    _fp32_attention_args((qkv, out, dout, dqkv, stats), (3 * T, T, T, 3 * T, B * n_heads * h * w * 3))
    code = _ATTN_CODE[attn_type] if isinstance(attn_type, str) else attn_type
    check(lib().kdb_attention_vjp(ptr(qkv), ptr(out), ptr(dout), ptr(dqkv), ptr(stats), B, h, w, n_heads, d_head, code, attn_param, shift,
                                   stream()))
    return dqkv


# ---------------------------------------------------------------------------------------------
# sample scoring (KID / FID)
# ---------------------------------------------------------------------------------------------

def _features(*tensors):
    for t in tensors:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError(f"features must be contiguous fp32 (got {t.dtype}, shape {tuple(t.shape)})")


@_on_device_of_first
def mmd_sums(x, y, x_offsets, y_offsets):
    """x [m, d] and y [n, d] contiguous fp32; x_offsets / y_offsets: S + 1 row bounds each (host ints), segment s pairing rows
    x_offsets[s]:x_offsets[s+1] of x with y_offsets[s]:y_offsets[s+1] of y -> [S, 4] float64 (k(x, x) off-diagonal sum, k(y, y)
    off-diagonal sum, k(x, y) sum, squared MMD) with the polynomial kernel (kdb_mmd_sums)."""
    require_cuda(x, y)
    _features(x, y)
    S = len(x_offsets) - 1
    if len(y_offsets) != S + 1 or x.shape[1] != y.shape[1]:
        raise ValueError(f"{len(x_offsets)} x bounds and {len(y_offsets)} y bounds; feature widths {x.shape[1]} and {y.shape[1]}")
    xo = (_i64 * (S + 1))(*x_offsets)
    yo = (_i64 * (S + 1))(*y_offsets)
    need = int(lib().kdb_mmd_workspace_bytes(xo, yo, S))
    if need < 0:
        check(need)
    ws = torch.empty(need, dtype=torch.uint8, device=x.device)
    out = torch.empty(S, 4, dtype=torch.float64, device=x.device)
    check(lib().kdb_mmd_sums(ptr(x), x.shape[0], ptr(y), y.shape[0], x.shape[1], xo, yo, S, ptr(out), ptr(ws), need, stream()))
    return out


@_on_device_of_first
def polynomial_kernel(x, y):
    """x [B, m, d] and y [B, n, d] contiguous fp32 -> [B, m, n] fp32 (x . y^T / d + 1)^3 (kdb_polynomial_kernel)."""
    require_cuda(x, y)
    _features(x, y)
    B, m, d = x.shape
    n = y.shape[1]
    out = torch.empty(B, m, n, dtype=torch.float32, device=x.device)
    check(lib().kdb_polynomial_kernel(ptr(x), ptr(y), ptr(out), B, m, n, d, stream()))
    return out


@_on_device_of_first
def feature_mean_cov(x):
    """x [n, d] contiguous fp32 -> (mean [d], cov [d, d]) fp32, x.mean(0) and torch.cov(x.T) (kdb_feature_mean_cov)."""
    require_cuda(x)
    _features(x)
    n, d = x.shape
    mean = torch.empty(d, dtype=torch.float32, device=x.device)
    cov = torch.empty(d, d, dtype=torch.float32, device=x.device)
    check(lib().kdb_feature_mean_cov(ptr(x), n, d, ptr(mean), ptr(cov), stream()))
    return mean, cov


# ---------------------------------------------------------------------------------------------
# training loop
# ---------------------------------------------------------------------------------------------

@_on_device_of_first
def ema_update(dsts, srcs, modes, weight):
    """kdb_ema_update: dst <- torch.lerp(dst, src, weight) (EMA_LERP) or dst <- src (EMA_COPY) for every (dst, src, mode), contiguous fp32
    tensors of equal size on one CUDA device, in one launch on the current stream."""
    require_cuda(*dsts, *srcs)
    table = (KdbEmaSeg * max(len(dsts), 1))()
    for i, (d, s, m) in enumerate(zip(dsts, srcs, modes)):
        table[i].src, table[i].dst, table[i].n, table[i].mode = s.data_ptr(), d.data_ptr(), d.numel(), m
    check(lib().kdb_ema_update(table, len(dsts), weight, stream()))


@_on_device_of_first
def augment(images, draws, a_prob, a_scale, a_aniso, a_trans, disable_all, with_mat=False):
    """kdb_augment: images [B, C, H, W] uint8 and draws [B, 13] fp32 on one CUDA device -> (image, image_orig, cond), with the matrices
    [B, 3, 3] appended when with_mat, fp32 on that device, in one launch on the current stream."""
    require_cuda(images, draws)
    if images.dtype != torch.uint8 or images.ndim != 4 or not images.is_contiguous():
        raise ValueError(f"images must be contiguous uint8 [B, C, H, W] (got {images.dtype}, shape {tuple(images.shape)})")
    B, C, H, W = images.shape
    if draws.dtype != torch.float32 or tuple(draws.shape) != (B, 13) or not draws.is_contiguous() or draws.device != images.device:
        raise ValueError(f"draws must be contiguous fp32 [{B}, 13] on {images.device} (got {draws.dtype}, shape {tuple(draws.shape)}, "
                         f"{draws.device})")
    image = torch.empty(B, C, H, W, dtype=torch.float32, device=images.device)
    image_orig = torch.empty_like(image)
    cond = torch.empty(B, 9, dtype=torch.float32, device=images.device)
    mat = torch.empty(B, 3, 3, dtype=torch.float32, device=images.device) if with_mat else None
    check(lib().kdb_augment(ptr(images), ptr(draws), B, C, H, W, a_prob, a_scale, a_aniso, a_trans, int(bool(disable_all)), ptr(image),
                            ptr(image_orig), ptr(cond), ptr(mat), stream()))
    return (image, image_orig, cond, mat) if with_mat else (image, image_orig, cond)
