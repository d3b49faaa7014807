"""The token-stream GEMM (gemm_wg_kernel) and the stand-alone attention kernels (attn_ws_kernel, attn_na_kernel) bit for bit: SHA-256
digests of their outputs against tests/golden/tc_digests.json.  These kernels share the TMA ring and named-barrier protocol of
csrc/tc_common.cuh with the fused level-0 kernels, whose digests test_gpu_fused_pipeline.py pins; a change of that protocol must leave
every result bit where it was.

The GEMM cases cover both tile widths (BN 128: 3 ring stages, BN 64: 4), an M tail, one k-block, fewer and more k-blocks than ring
stages, fewer tiles than SMs and an uneven number of tiles per CTA, and the GEGLU epilogue with and without the fused RMSNorm.  The
attention cases cover windows with both shifts and an odd window count, global attention over 1, 2 and 16 key blocks and the
neighbourhood kernel, each with and without the logit bound.  One bf16 Engine.forward of the cfg2 model at 64x64 (batch 3) on the
shared and on the per-sample conditioning route runs the GEMM's RESID, SPLIT, QKV_ROPE, merge and PATCHOUT epilogues.  Every output
buffer starts as NaN, so an element left unwritten changes the digest and fails the finiteness check.

Record the golden (on the build whose results are the reference):  python tests/test_gpu_tc_digests.py --record OUT.json
"""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
GOLDEN = ROOT / "tests" / "golden" / "tc_digests.json"
DEV = "cuda"
SCALE = 10.0            # |q . k| bound of the attention inputs

# (M, N, K): BN = 128 when N % 128 == 0, else 64
GEMM_CASES = [
    (256, 256, 64),                          # BN 128, one k-block
    (200, 192, 128),                         # BN 64, M tail, 2 k-blocks < 4 stages
    (1000, 384, 512),                        # BN 128, M tail, 8 k-blocks > 3 stages
    (128 * 40, 320, 320),                    # BN 64, 5 k-blocks > 4 stages
    (256, 128, 256),                         # 2 tiles: fewer than SMs
    ((132 * 2 + 5) * 128, 128, 192),         # uneven tiles per CTA, k-blocks = stages
]
# (M, F, K, fused RMSNorm)
GEGLU_CASES = [(1000, 256, 256, False), (1000, 256, 256, True), ((132 * 2 + 5) * 128, 128, 128, True)]
# (kind, B, h, w, nh, shift)
ATTN_CASES = [
    ("shifted-window", 1, 8, 24, 2, 0),      # 3 windows
    ("shifted-window", 3, 24, 8, 4, 4),      # 9 windows, both seams
    ("global", 2, 8, 16, 2, 0),              # 1 key block
    ("global", 3, 16, 16, 2, 0),             # 2 key blocks
    ("global", 1, 32, 64, 3, 0),             # 16 key blocks
    ("neighborhood", 2, 16, 32, 2, 0),
]
ROUTES = ["shared", "per_sample"]


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _nan(shape, dtype=torch.bfloat16):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _written(out):
    assert bool(torch.isfinite(out.float()).all()), "an output element was not written"
    return _digest(out)


def run_gemm(M, N, K):
    from k_diffusion import _native as N_
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).to(DEV)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(torch.bfloat16).to(DEV)
    out = _nan((M, N))
    N_.check(N_.lib().kdb_gemm_bf16(N_.ptr(a), N_.ptr(w), N_.ptr(out), M, N, K, N_.stream()))
    torch.cuda.synchronize()
    return _written(out)


def run_geglu(M, F, K, norm):
    from k_diffusion import _native as N_
    g = torch.Generator().manual_seed(M + F + K)
    x = (torch.randn(M, K, generator=g) * (0.5 + torch.rand(M, 1, generator=g) * 3)).to(torch.bfloat16)
    w_up = (torch.randn(2 * F, K, generator=g) / K ** 0.5).to(torch.bfloat16)
    ss = None
    if norm:        # sum(x^2) per 128-channel slot of [M, 8]; the unused slots NaN: they must never be read
        ss = torch.full((M, 8), float("nan"))
        ss[:, :K // 128] = x.double().pow(2).view(M, K // 128, 128).sum(2).float()
        ss = ss.to(DEV)
    out = _nan((M, F))
    w_il = N_.interleave_geglu_rows(w_up.to(DEV))
    N_.check(N_.lib().kdb_gemm_bf16_geglu(N_.ptr(x.to(DEV)), N_.ptr(w_il), N_.ptr(out), M, 2 * F, K, N_.ptr(ss), N_.stream()))
    torch.cuda.synchronize()
    return _written(out)


def run_attn(kind, B, h, w, nh, shift, bounded):
    from k_diffusion import _native as N_
    g = torch.Generator().manual_seed(B * 1000 + h * 10 + w + nh + shift)
    t = torch.randn(B, h * w, 3, nh, 64, generator=g)
    t[:, :, :2] = t[:, :, :2] / t[:, :, :2].norm(dim=-1, keepdim=True) * SCALE ** 0.5
    qkv = t.to(torch.bfloat16).reshape(B, h * w, 3 * nh * 64).to(DEV)
    bound = torch.full((nh,), SCALE, device=DEV) if bounded else None
    param = {"shifted-window": 8, "neighborhood": 7, "global": 0}[kind]
    out = _nan((B, h * w, nh * 64))
    N_.check(N_.lib().kdb_attention(N_.PREC_BF16, 1, N_.ptr(qkv), N_.ptr(out), B, h, w, nh, 64, N_._ATTN_CODE[kind], param, shift,
                                    N_.ptr(bound), N_.stream()))
    torch.cuda.synchronize()
    return _written(out)


def run_engine(route):
    from k_diffusion import _native as N_
    from test_gpu_bf16_stages import CONFIGS, latent, make
    raw_fn, H, W, sigmas, _ = CONFIGS["cfg2_64_b3"]
    inner, P = make(raw_fn(), H, W)
    eng = inner.to(DEV).eval().engine()
    sigma = torch.tensor(sigmas)
    img, s_d = latent(7, len(sigmas), H, W, sigma).to(DEV), sigma.to(DEV)
    shared = route == "shared"
    table, stride = eng.conditioning(s_d[:1] if shared else s_d), 0 if shared else eng.cond_stride
    out = _nan(img.shape, img.dtype)
    eng.forward(img, s_d, table, stride, P.sigma_data, N_.PREC_BF16, out=out)
    torch.cuda.synchronize()
    return _written(out)


def _key(*case):
    return " ".join(str(c) for c in case)


def _all_cases():
    yield from ((_key("gemm", *c), run_gemm, c) for c in GEMM_CASES)
    yield from ((_key("geglu", *c), run_geglu, c) for c in GEGLU_CASES)
    yield from ((_key("attn", *c, b), run_attn, c + (b,)) for c in ATTN_CASES for b in (False, True))
    yield from ((_key("engine cfg2_64_b3", r), run_engine, (r,)) for r in ROUTES)


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", GEMM_CASES)
def test_gemm_digests(golden, M, N, K):
    assert run_gemm(M, N, K) == golden[_key("gemm", M, N, K)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,F,K,norm", GEGLU_CASES)
def test_gemm_geglu_digests(golden, M, F, K, norm):
    assert run_geglu(M, F, K, norm) == golden[_key("geglu", M, F, K, norm)]


@pytest.mark.gpu
@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("kind,B,h,w,nh,shift", ATTN_CASES)
def test_attention_digests(golden, kind, B, h, w, nh, shift, bounded):
    assert run_attn(kind, B, h, w, nh, shift, bounded) == golden[_key("attn", kind, B, h, w, nh, shift, bounded)]


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
def test_engine_forward_digests(golden, route):
    assert run_engine(route) == golden[_key("engine cfg2_64_b3", route)]


if __name__ == "__main__":
    assert len(sys.argv) == 3 and sys.argv[1] == "--record", __doc__
    rec = {}
    for key, fn, args in _all_cases():
        rec[key] = fn(*args)
        assert fn(*args) == rec[key], f"{key}: two runs differ"
    Path(sys.argv[2]).write_text(json.dumps(rec, indent=1) + "\n")
    print(f"recorded {len(rec)} digests -> {sys.argv[2]}")
