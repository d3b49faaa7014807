"""ctypes binding of libkdb200.so (C ABI declared in include/kdiffusion_b200.h).

There is deliberately NO fallback: if the shared library is missing or a tensor is not on a CUDA
device the call raises.  PyTorch is used only for device memory, streams and views.
"""
import contextlib
import ctypes
import math
import functools
import os
from pathlib import Path

import torch

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("KDB200_LIB", _HERE / "_lib" / "libkdb200.so"))

PREC_FP32, PREC_BF16 = 0, 1
ATTN_NONE, ATTN_GLOBAL, ATTN_NEIGHBORHOOD, ATTN_SHIFTED_WINDOW = 0, 1, 2, 3
MAX_LEVELS = 8
ABI_VERSION = 7

_vp, _i32, _i64, _f32, _f64, _u64, _sz = (ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double,
                                           ctypes.c_uint64, ctypes.c_size_t)


class KdbModelConfig(ctypes.Structure):
    _fields_ = [
        ("n_levels", _i32), ("in_channels", _i32), ("out_channels", _i32), ("patch_h", _i32), ("patch_w", _i32),
        ("mapping_width", _i32), ("mapping_depth", _i32), ("mapping_d_ff", _i32), ("num_classes", _i32), ("mapping_cond_dim", _i32),
        ("width", _i32 * MAX_LEVELS), ("depth", _i32 * MAX_LEVELS), ("d_ff", _i32 * MAX_LEVELS), ("attn_type", _i32 * MAX_LEVELS),
        ("d_head", _i32 * MAX_LEVELS), ("attn_param", _i32 * MAX_LEVELS),
    ]


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
    "kdb_model_debug_tap": (_i32, [_vp, ctypes.c_char_p, _vp, _i64]),
    "kdb_model_tap_count": (_i64, [_vp]),
    "kdb_gemm_bf16": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "kdb_gemm_bf16_geglu": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "kdb_ffn_fused_bf16": (_i32, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "kdb_attention": (_i32, [_i32, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
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


class Engine:
    """Owns one KdbModel handle for one ImageTransformerDenoiserModelV2 instance on one device."""

    def __init__(self, spec):
        cfg = KdbModelConfig()
        levels = spec["levels"]
        if len(levels) > MAX_LEVELS:
            raise ValueError(f"at most {MAX_LEVELS} levels supported")
        cfg.n_levels = len(levels)
        cfg.in_channels, cfg.out_channels = spec["in_channels"], spec["out_channels"]
        cfg.patch_h, cfg.patch_w = spec["patch_size"]
        cfg.mapping_width, cfg.mapping_depth, cfg.mapping_d_ff = spec["mapping_width"], spec["mapping_depth"], spec["mapping_d_ff"]
        cfg.num_classes, cfg.mapping_cond_dim = spec["num_classes"], spec["mapping_cond_dim"]
        for i, lv in enumerate(levels):
            cfg.width[i], cfg.depth[i], cfg.d_ff[i] = lv["width"], lv["depth"], lv["d_ff"]
            cfg.attn_type[i] = _ATTN_CODE[lv["attn"]]
            cfg.d_head[i] = lv.get("d_head", 0)
            cfg.attn_param[i] = lv.get("attn_param", 0)
        self.cfg = cfg
        self._h = _vp()
        check(lib().kdb_model_create(ctypes.byref(cfg), ctypes.byref(self._h)))
        self._sig = None
        self._held = {}
        self._ws = None
        self._stride = None
        self.device = None

    def __del__(self):
        try:
            if getattr(self, "_h", None) and _lib is not None:
                _lib.kdb_model_destroy(self._h)
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
                check(lib().kdb_model_set_tensor(self._h, k.encode(), ptr(t32), shape, t32.ndim))
            check(lib().kdb_model_finalize(self._h, stream()))
        self._held = held
        self._sig = sig
        self._stride = int(lib().kdb_model_cond_stride(self._h))

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

    def _workspace(self, precision, B, H, W, device):
        need = int(lib().kdb_model_workspace_bytes(self._h, precision, B, H, W))
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=device)
        return self._ws

    def forward(self, x, sigma, cond, cond_batch_stride, sigma_data, precision, out=None):
        """x [B,C,H,W] fp32; sigma [B]; cond rows; sigma_data <= 0 -> raw inner model."""
        B, _, H, W = x.shape
        if out is None:
            out = torch.empty(B, self.cfg.out_channels, H, W, device=x.device, dtype=torch.float32)
        ws = self._workspace(precision, B, H, W, x.device)
        with device_of(x):
            check(lib().kdb_model_forward(self._h, precision, B, H, W, ptr(x), ptr(sigma), float(sigma_data), ptr(cond), cond_batch_stride,
                                          ptr(out), ptr(ws), ws.numel(), stream()))
        return out

    def arm_tap(self, name, capacity, device):
        buf = torch.empty(capacity, dtype=torch.float32, device=device)
        check(lib().kdb_model_debug_tap(self._h, name.encode(), ptr(buf), capacity))
        return buf

    def tap_count(self):
        return int(lib().kdb_model_tap_count(self._h))


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
