"""The token-stream GEMM's GEGLU and TokenSplit epilogues bit for bit at the shapes the benchmark runs them at: SHA-256 digests against
tests/golden/gemm_epilogue_digests.json, recorded on the build before the GEGLU epilogue moved onto the accumulator fragments and the TokenSplit
epilogue onto TMA.  Every epilogue formula and accumulation order was kept, so every bit must stay where it was.

The GEGLU GEMM (kdb_gemm_bf16_geglu) runs at the cfg2 and cfg5 up_proj shapes, with and without the fused RMSNorm, and at an M that is
not a multiple of 128.  One bf16 Engine.forward at cfg2's full shape (B = 32, 256 x 256) and one at cfg5's shape (512 x 512, B = 2), on
the shared conditioning route, are tapped after both TokenSplits, after the GEGLU of a level-1 and of a middle-level layer, and at the
output; so is one at 64 x 384, whose splits scatter per thread (their 128-row blocks are no TMA box).

Record the golden (on the build whose results are the reference):  python tests/test_gpu_gemm_epilogue_bits.py --record OUT.json
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
from test_gpu_tc_digests import _written, run_geglu  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "gemm_epilogue_digests.json"
DEV = "cuda"

# (M, F, K, fused RMSNorm): up_proj of cfg2 (B = 32) levels 1 and middle, cfg5 (B = 16) levels 0, 1 and middle, and an M tail
GEGLU_CASES = [(M, F, K, norm) for (M, F, K) in [(32768, 768, 256), (8192, 1536, 512), (262144, 768, 256), (65536, 1536, 512),
                                                 (16384, 3072, 1024), (5000, 1536, 512)] for norm in (False, True)]
# layer 2: the first level-1 layer, layer 5: a middle-level layer (depths 2, 2, 4)
TAPS = ["L0.split", "L1.split", "layer2.geglu", "layer5.geglu", "out"]


def cfg5_raw():
    return {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [512, 512], "patch_size": [4, 4],
                      "depths": [2, 2, 4], "widths": [256, 512, 1024], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160}}


# name: (raw config, H, W, batch)
ENGINES = {
    "cfg2_256_b32": (lambda: cfg2_raw(256, 256), 256, 256, 32),
    "cfg5_512_b2": (cfg5_raw, 512, 512, 2),
    # coarse grids 48 and 24 tokens wide: no 128-row block is a quadrant box, both splits take the per-thread scatter
    "cfg2_64x384_b2": (lambda: cfg2_raw(64, 384), 64, 384, 2),
}
_engines = {}


def _engine(name):
    """(engine, input, sigma, conditioning table, sigma_data) of one config, built once per process"""
    if name not in _engines:
        raw_fn, H, W, B = ENGINES[name]
        inner, P = make(raw_fn(), H, W)
        eng = inner.to(DEV).eval().engine()
        sigma = torch.linspace(0.3, 40.0, B)
        img = latent(7, B, H, W, sigma).to(DEV)
        s_d = sigma.to(DEV)
        _engines[name] = (eng, img, s_d, eng.conditioning(s_d[:1]), P.sigma_data)
    return _engines[name]


def run_tap(name, tap):
    from k_diffusion import _native as N_
    eng, img, s_d, table, sd_ = _engine(name)
    if tap == "out":
        out = eng.forward(img, s_d, table, 0, sd_, N_.PREC_BF16)
        torch.cuda.synchronize()
        return _written(out)
    cap = 1 << 25                            # the largest tap, cfg2's layer2.geglu, has 32 x 32 x 32 x 768 elements
    buf = eng.arm_tap(tap, cap, DEV)
    buf.fill_(float("nan"))
    eng.forward(img, s_d, table, 0, sd_, N_.PREC_BF16)
    torch.cuda.synchronize()
    n = eng.tap_count()
    assert 0 < n <= cap, f"tap {tap}: {n} elements"
    return _written(buf[:n])


def _key(*case):
    return " ".join(str(c) for c in case)


def _all_cases():
    yield from ((_key("geglu", *c), run_geglu, c) for c in GEGLU_CASES)
    yield from ((_key("engine", e, t), run_tap, (e, t)) for e in ENGINES for t in TAPS)


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("M,F,K,norm", GEGLU_CASES)
def test_geglu_gemm_bits(golden, M, F, K, norm):
    assert run_geglu(M, F, K, norm) == golden[_key("geglu", M, F, K, norm)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("tap", TAPS)
@pytest.mark.parametrize("engine", list(ENGINES))
def test_engine_epilogue_bits(golden, engine, tap):
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
