"""The token-stream GEMM (gemm_wg_kernel) at the edges of its row-block schedule, for every epilogue, with every output fenced: M <= 128
(one row block, partly past M); an odd number of row blocks whose last one is a tail; fewer tiles than SMs; 273 tiles, which 132 CTAs
share unevenly; both tile widths.  SHA-256 digests of every output against tests/golden/gemm_edge_digests.json.  Every
output starts as NaN (an element left unwritten fails the finiteness check) and is followed by a sentinel region that must come out
untouched, so a store of a row past M shows.

The STORE and GEGLU epilogues run through kdb_gemm_bf16 / kdb_gemm_bf16_geglu.  RESID, QKV_ROPE, GEGLU with the fused RMSNorm, the
TokenMerge gather through the 5-D A box, the TokenSplit through its TMA boxes and per thread, and PATCH_OUT run inside bf16
Engine.forward calls whose levels have an odd number of row blocks (and a middle level of one row block), tapped after each such GEMM;
the forward's output image (PATCH_OUT) is written into a buffer with a sentinel behind it.

Record the golden (on the build whose results are the reference):  python tests/test_gpu_gemm_edges.py --record OUT.json
"""
import json
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200"), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
from test_gpu_bf16_stages import cfg2_raw, latent, make  # noqa: E402
from test_gpu_tc_digests import _digest  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "gemm_edge_digests.json"
DEV = "cuda"
SENTINEL = 4096          # elements after every output
SENTINEL_BITS = 0x5A5A   # bf16 / the low half of an fp32 element, never a result here

# (M, N, K); BN = 128 when N % 128 == 0, else 64.  Row blocks: ceil(M / 128)
STORE_CASES = [
    (100, 256, 128),             # one row block, partly past M; 2 tiles: fewer than SMs
    (128, 192, 64),              # the same at BN 64, M exactly one block
    (128 * 5 - 3, 256, 256),     # 5 row blocks, the last one a tail
    (128 * 7, 192, 320),         # 7 row blocks at BN 64, 5 k-blocks
    (128 * 273 - 5, 64, 128),    # 273 tiles (3 x 7 x 13) at BN 64, the last row block a tail
    (128 * 273, 128, 192),       # 273 tiles at BN 128, k-blocks = ring stages
]
# (M, F, K, fused RMSNorm)
GEGLU_CASES = [(77, 256, 256, True), (128 * 5 - 3, 768, 512, False), (128 * 5 - 3, 768, 512, True)]


def sw_global_raw(H, W):
    """a shifted-window level 0 (C = 128) over a global level 1 (C = 256): any level-0 grid whose sides are multiples of 8"""
    return {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [H, W], "patch_size": [4, 4],
                      "depths": [1, 1], "widths": [128, 256], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160,
                      "self_attns": [{"type": "shifted-window", "d_head": 64, "window_size": 8}, {"type": "global", "d_head": 64}]}}


L1 = [f"layer2.{s}" for s in ("qkv", "ao", "geglu", "ff")]   # the first level-1 layer of cfg2 (depths 2, 2, 4)
MID = [f"layer5.{s}" for s in ("qkv", "ao", "geglu", "ff")]  # a middle-level layer
# name: (raw config, H, W, batch, taps)
ENGINES = {
    # level 1: 8 x 16 tokens x 3 = 3 row blocks, merge 0 and split 0 through 5-D boxes of 8 x 16 coarse tokens; middle level: 96 tokens,
    # one row block, merge 1 and split 1 through boxes of 16 x 8
    "cfg2_64x128_b3": (lambda: cfg2_raw(64, 128), 64, 128, 3, L1 + MID + ["L0.merge", "L1.merge", "L0.split", "L1.split"]),
    # level 1: 8 x 48 tokens = 3 row blocks, coarse grids 48 and 24 wide: both splits scatter per thread
    "cfg2_64x384_b1": (lambda: cfg2_raw(64, 384), 64, 384, 1, L1 + MID + ["L0.split", "L1.split"]),
    # level 0: 8 x 40 tokens = 3 row blocks (PATCH_OUT, the GEGLU left to the generic GEMM: M % 128 != 0); level 1: 80 tokens
    "swg_32x160_b1": (lambda: sw_global_raw(32, 160), 32, 160, 1, ["layer0.geglu", "layer0.ff", "layer1.qkv", "layer1.ao", "layer1.geglu",
                                                                      "layer1.ff", "L0.merge", "L0.split"]),
}
_engines = {}


def _buffer(n, dtype):
    """n NaN elements followed by the sentinel region, as one allocation"""
    buf = torch.full((n + SENTINEL,), float("nan"), dtype=dtype, device=DEV)
    bits = buf.view(torch.int16) if dtype == torch.bfloat16 else buf.view(torch.int32)
    bits[n * (bits.numel() // buf.numel()):] = SENTINEL_BITS
    return buf


def _checked(buf, n):
    """digest of the first n elements; asserts that all were written and that the sentinel region after them was not"""
    bits = buf.view(torch.int16) if buf.dtype == torch.bfloat16 else buf.view(torch.int32)
    tail = bits[n * (bits.numel() // buf.numel()):]
    assert bool((tail == SENTINEL_BITS).all()), f"{int((tail != SENTINEL_BITS).sum())} elements written past the output"
    out = buf[:n]
    assert bool(torch.isfinite(out.float()).all()), "an output element was not written"
    return _digest(out)


def run_store(M, N, K):
    from k_diffusion import _native as N_
    g = torch.Generator().manual_seed(M * 5 + N * 3 + K)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).to(DEV)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(torch.bfloat16).to(DEV)
    buf = _buffer(M * N, torch.bfloat16)
    N_.check(N_.lib().kdb_gemm_bf16(N_.ptr(a), N_.ptr(w), N_.ptr(buf), M, N, K, N_.stream()))
    torch.cuda.synchronize()
    return _checked(buf, M * N)


def run_geglu(M, F, K, norm):
    from k_diffusion import _native as N_
    g = torch.Generator().manual_seed(M + 3 * F + K)
    x = (torch.randn(M, K, generator=g) * (0.5 + torch.rand(M, 1, generator=g) * 3)).to(torch.bfloat16)
    w_up = (torch.randn(2 * F, K, generator=g) / K ** 0.5).to(torch.bfloat16)
    ss = None
    if norm:        # sum(x^2) per 128-channel slot of [M, 8]; the unused slots NaN: they must never be read
        ss = torch.full((M, 8), float("nan"))
        ss[:, :K // 128] = x.double().pow(2).view(M, K // 128, 128).sum(2).float()
        ss = ss.to(DEV)
    buf = _buffer(M * F, torch.bfloat16)
    w_il = N_.interleave_geglu_rows(w_up.to(DEV))
    N_.check(N_.lib().kdb_gemm_bf16_geglu(N_.ptr(x.to(DEV)), N_.ptr(w_il), N_.ptr(buf), M, 2 * F, K, N_.ptr(ss), N_.stream()))
    torch.cuda.synchronize()
    return _checked(buf, M * F)


def _engine(name):
    """(engine, input, sigma, conditioning table, sigma_data, B, H, W) of one config, built once per process"""
    if name not in _engines:
        raw_fn, H, W, B, _ = ENGINES[name]
        inner, P = make(raw_fn(), H, W)
        eng = inner.to(DEV).eval().engine()
        sigma = torch.linspace(0.3, 40.0, B)
        img = latent(11, B, H, W, sigma).to(DEV)
        s_d = sigma.to(DEV)
        _engines[name] = (eng, img, s_d, eng.conditioning(s_d[:1]), P.sigma_data, B, H, W)
    return _engines[name]


def run_tap(name, tap):
    from k_diffusion import _native as N_
    eng, img, s_d, table, sd_, B, H, W = _engine(name)
    n = B * 3 * H * W
    out = _buffer(n, torch.float32)
    if tap != "out":
        cap = B * H * W * 64                  # the largest tap, a level-0 GEGLU, has B x H / 4 x W / 4 x 384 elements
        buf = eng.arm_tap(tap, cap, DEV)
        buf.fill_(float("nan"))
    eng.forward(img, s_d, table, 0, sd_, N_.PREC_BF16, out=out[:n].view(B, 3, H, W))
    torch.cuda.synchronize()
    digest = _checked(out, n)
    if tap == "out":
        return digest
    k = eng.tap_count()
    assert 0 < k <= cap, f"tap {tap}: {k} elements"
    out_t = buf[:k]
    assert bool(torch.isfinite(out_t).all()), f"tap {tap}: an element was not written"
    return _digest(out_t)


def _key(*case):
    return " ".join(str(c) for c in case)


ENGINE_CASES = [(e, t) for e, spec in ENGINES.items() for t in spec[4] + ["out"]]


def _all_cases():
    yield from ((_key("store", *c), run_store, c) for c in STORE_CASES)
    yield from ((_key("geglu", *c), run_geglu, c) for c in GEGLU_CASES)
    yield from ((_key("engine", *c), run_tap, c) for c in ENGINE_CASES)


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", STORE_CASES)
def test_edge_store_bits(golden, M, N, K):
    assert run_store(M, N, K) == golden[_key("store", M, N, K)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,F,K,norm", GEGLU_CASES)
def test_edge_geglu_bits(golden, M, F, K, norm):
    assert run_geglu(M, F, K, norm) == golden[_key("geglu", M, F, K, norm)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("engine,tap", ENGINE_CASES)
def test_edge_engine_bits(golden, engine, tap):
    assert run_tap(engine, tap) == golden[_key("engine", engine, tap)]


if __name__ == "__main__":
    assert len(sys.argv) == 3 and sys.argv[1] == "--record", __doc__
    rec = {}
    for key, fn, args in _all_cases():
        rec[key] = fn(*args)
        assert fn(*args) == rec[key], f"{key}: two runs differ"
        print(key, rec[key][:16], flush=True)
    Path(sys.argv[2]).write_text(json.dumps(rec, indent=1) + "\n")
    print(f"recorded {len(rec)} digests -> {sys.argv[2]}")
