"""Tensor-core (wgmma/TMA) kernels against a plain PyTorch fp32 reference of the same op."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (128, 64, 64), (256, 384, 128), (8192, 768, 128), (1000, 256, 512),
                                   (2048, 512, 1536), (196, 768, 256), (4096, 1024, 2048), (32768, 128, 384),
                                   # K = 128 with several n-blocks and M not a multiple of the tile
                                   (65536, 768, 128), (40000, 384, 128), (20000, 256, 128), (300, 768, 128), (33000, 512, 128)])
def test_gemm_bf16_tcgen05(M, N, K):
    from k_diffusion import _native as N_
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
    got = N_.gemm_bf16(a, w).float()
    want = a.float() @ w.float().T
    err = (got - want).abs()
    tol = 1e-2 * want.abs() + 2e-2           # one bf16 ulp of the output (2^-8 relative) + accumulation-order slack
    assert bool((err <= tol).all()), f"max err {float(err.max()):.4f} at {int(err.argmax())}, want {float(want.flatten()[err.argmax()]):.4f}"
    # not a trivially-zero result
    assert float(got.abs().mean()) > 0.1


def test_gemm_k_order_and_row_identity():
    """A = row-selector, W = distinct rows: catches swizzle / descriptor-advance mistakes exactly."""
    from k_diffusion import _native as N_
    K, N, M = 256, 128, 256
    a = torch.zeros(M, K, device=DEV, dtype=torch.bfloat16)
    idx = torch.arange(M, device=DEV) % K
    a[torch.arange(M, device=DEV), idx] = 1.0
    w = ((torch.arange(N, device=DEV)[:, None] * 0.5 + torch.arange(K, device=DEV)[None, :] * 0.25) % 61 - 30).to(torch.bfloat16)
    got = N_.gemm_bf16(a, w).float()
    want = w.float().T[idx]                   # row m of C = column idx[m] of W^T
    assert torch.equal(got, want)


def _qkv(B, h, w, nh, seed):
    """qkv [B, h*w, 3*nh*64] bf16 with cosine-normalised q,k (|q| = |k| = sqrt(10)) like the real layer input."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    t = torch.randn(B, h * w, 3, nh, 64, device=DEV, generator=g)
    t[:, :, :2] = t[:, :, :2] / t[:, :, :2].norm(dim=-1, keepdim=True) * 10 ** 0.5
    return t.to(torch.bfloat16).reshape(B, h * w, 3 * nh * 64)


def _ref_attention(qkv, h, w, nh, kind, param, shift):
    from oracle import kdiff_oracle as O
    B = qkv.shape[0]
    q, k, v = qkv.float().cpu().view(B, h, w, 3, nh, 64).unbind(3)
    if kind == "global":
        o = O.global_attention(q, k, v)
    elif kind == "shifted-window":
        o = O.shifted_window_attention(q, k, v, param, shift)
    else:
        o = O.neighborhood_attention(q, k, v, param)
    return o.reshape(B, h * w, nh * 64)


@pytest.mark.parametrize("B,h,w,nh,kind,param,shift", [
    (2, 16, 16, 2, "shifted-window", 8, 0), (2, 16, 16, 2, "shifted-window", 8, 4), (1, 8, 8, 4, "shifted-window", 8, 4),
    (3, 64, 64, 2, "shifted-window", 8, 4), (2, 32, 24, 4, "shifted-window", 8, 0),
    (2, 16, 16, 8, "global", 0, 0), (1, 8, 16, 2, "global", 0, 0), (1, 32, 32, 4, "global", 0, 0), (2, 16, 24, 1, "global", 0, 0),
    (2, 16, 32, 2, "neighborhood", 7, 0), (1, 64, 64, 2, "neighborhood", 7, 0), (2, 32, 32, 4, "neighborhood", 7, 0),
    (1, 24, 48, 1, "neighborhood", 7, 0), (1, 16, 112, 3, "neighborhood", 7, 0)])
def test_attention_tcgen05_vs_reference(B, h, w, nh, kind, param, shift):
    from k_diffusion import _native as N_
    qkv = _qkv(B, h, w, nh, seed=h * w + nh + shift)
    want = _ref_attention(qkv, h, w, nh, kind, param, shift)
    slow = N_.attention(qkv, h, w, nh, 64, kind, param, shift, fast=False).float().cpu()
    fast = N_.attention(qkv, h, w, nh, 64, kind, param, shift, fast=True).float().cpu()
    # bf16 output (2^-8 relative) + bf16 P inside the tensor-core path
    for name, got in (("generic", slow), ("tensor core", fast)):
        err = (got - want).abs()
        assert float(err.max()) < 3e-2 and float(err.mean()) < 3e-3, f"{name}: max {float(err.max()):.4f} mean {float(err.mean()):.5f}"


@pytest.mark.parametrize("B,h,w,nh,kind,param,shift", [
    (2, 16, 16, 2, "shifted-window", 8, 0), (3, 64, 64, 2, "shifted-window", 8, 4), (1, 8, 8, 4, "shifted-window", 8, 4),
    (2, 16, 16, 8, "global", 0, 0), (3, 16, 16, 8, "global", 0, 0), (1, 8, 16, 2, "global", 0, 0), (2, 32, 32, 4, "global", 0, 0),
    (1, 32, 32, 16, "global", 0, 0), (5, 16, 32, 3, "global", 0, 0), (32, 16, 16, 8, "global", 0, 0),
    (2, 16, 32, 2, "neighborhood", 7, 0), (1, 64, 64, 2, "neighborhood", 7, 0), (2, 32, 32, 4, "neighborhood", 7, 0),
    # large batches, odd tile counts
    (32, 64, 64, 2, "shifted-window", 8, 4), (32, 64, 64, 2, "shifted-window", 8, 0), (20, 32, 32, 4, "shifted-window", 8, 4),
    (8, 64, 64, 2, "neighborhood", 7, 0), (6, 32, 32, 4, "neighborhood", 7, 0), (3, 24, 48, 1, "neighborhood", 7, 0),
    (1, 16, 112, 3, "neighborhood", 7, 0), (1, 8, 8, 2, "shifted-window", 8, 4)])
def test_attention_tcgen05_bounded_softmax(B, h, w, nh, kind, param, shift):
    """Fixed-shift softmax (logit_bound = the cosine-similarity scale): single-pass kernels, at batch sizes up to 32, against the same
    oracle and tolerance as the row-maximum kernels."""
    from k_diffusion import _native as N_
    qkv = _qkv(B, h, w, nh, seed=h * w + nh + shift + 1)
    want = _ref_attention(qkv[:4], h, w, nh, kind, param, shift)
    bound = torch.full([nh], 10.0, device=DEV)
    fast = N_.attention(qkv, h, w, nh, 64, kind, param, shift, fast=True, logit_bound=bound)
    torch.cuda.synchronize()
    err = (fast[:4].float().cpu() - want).abs()
    assert float(err.max()) < 3e-2 and float(err.mean()) < 3e-3, f"max {float(err.max()):.4f} mean {float(err.mean()):.5f}"
    if B > 4:          # images beyond the oracle's slice: compare with the row-maximum kernel
        slow = N_.attention(qkv, h, w, nh, 64, kind, param, shift, fast=True)
        assert float((fast.float() - slow.float()).abs().max()) < 2e-2
    # a looser bound (scale 20 on the same data) must give the same softmax: shift invariance
    loose = N_.attention(qkv, h, w, nh, 64, kind, param, shift, fast=True, logit_bound=bound * 2)
    assert float((loose.float() - fast.float()).abs().max()) < 2e-2


def test_attention_generic_fp32_exact():
    from k_diffusion import _native as N_
    for kind, param, shift, h, w in (("global", 0, 0, 7, 7), ("shifted-window", 4, 2, 8, 12), ("neighborhood", 7, 0, 9, 12), ("neighborhood", 3, 0, 5, 4)):
        qkv = _qkv(2, h, w, 2, seed=h + w).float()
        want = _ref_attention(qkv, h, w, 2, kind, param, shift)
        got = N_.attention(qkv, h, w, 2, 64, kind, param, shift).cpu()
        assert float((got - want).abs().max()) < 2e-5, kind


@pytest.mark.parametrize("M,F", [(128, 192), (1280, 384), (148 * 128 * 2 + 384, 384), (131072, 384), (4096, 512)])
def test_ffn_fused_matches_reference_and_unfused_kernels(M, F):
    """tc_ffn_fused.cuh: x <- x + (value * gelu(gate))(x / rms) @ Wdown^T in one kernel, against (a) an fp32 torch reference of the same
    op and (b) the two stand-alone tensor-core kernels it replaces (within bf16 rounding of the output)."""
    from k_diffusion import _native as N_
    g = torch.Generator(device=DEV).manual_seed(M + F)
    C = 128
    x = (torch.randn(M, C, device=DEV, generator=g) * (0.5 + torch.rand(M, 1, device=DEV, generator=g) * 3)).to(torch.bfloat16)
    w_up = (torch.randn(2 * F, C, device=DEV, generator=g) / C ** 0.5).to(torch.bfloat16)
    w_dn = (torch.randn(C, F, device=DEV, generator=g) / F ** 0.5).to(torch.bfloat16)
    ss = torch.zeros(M, 8, device=DEV)
    ss[:, 0] = x.float().pow(2).sum(1)
    ss[:, 1:] = float("nan")                   # only slot 0 belongs to a 128-wide level: the others must never be read
    # (b) the stand-alone kernels
    h = N_.gemm_bf16_geglu(x, w_up, ss_in=ss)
    y_unfused = (x.float() + N_.gemm_bf16(h, w_dn).float()).to(torch.bfloat16)
    # (a) fp32 reference, hidden rounded to bf16 where the kernels round it
    xn = x.float() * torch.rsqrt(ss[:, :1] / C + 1e-6)
    u = xn @ w_up.float().T
    hid = (u[:, :F] * torch.nn.functional.gelu(u[:, F:])).to(torch.bfloat16).float()
    want = x.float() + hid @ w_dn.float().T
    ss_out = torch.full((M, 8), -1.0, device=DEV)
    got = N_.ffn_fused_bf16(x.clone(), w_up, w_dn, ss, ss_out)
    torch.cuda.synchronize()
    err = (got.float() - want).abs()
    tol = 1.5e-2 * want.abs() + 3e-2
    assert bool((err <= tol).all()), f"vs fp32 reference: max err {float(err.max()):.4f} (want {float(want.flatten()[err.argmax()]):.4f})"
    d = (got.float() - y_unfused.float()).abs()
    # (the stand-alone pair rounds the down projection to bf16 before the residual add, the fused kernel adds in fp32: one-ulp differences)
    assert bool((d <= 2 ** -6 * (want.abs() + 1.0)).all()), f"vs stand-alone kernels: max |diff| {float(d.max()):.4g}"
    # row statistics of the new stream for the next fused RMSNorm: slot 0 only
    want_ss = got.float().pow(2).sum(1)
    assert torch.allclose(ss_out[:, 0], want_ss, rtol=2e-2, atol=1e-2)
    assert bool((ss_out[:, 1:] == -1.0).all())
