"""Which kernels the engine launches for one forward, case by case.

The numerical tests accept every route the engine can take: a stage that moved off attn_block or ffn_fused onto the three-launch
path, or lost its fused RMSNorm, still passes them.  Here the sequence of launch families of one Engine.forward is compared with
tests/golden/engine_routes.json.  Families are coarse (attn_block, ffn_fused and every wgmma GEMM count as gemm_tc), but each route
choice shows in the sequence: one gemm_tc launch against gemm_tc, attn_tc, gemm_tc; rmsnorm present or absent; qknorm_rope present or
absent; rmsnorm before patch_out or not.

Cases:
  <config>/<route>  every configuration of test_gpu_bf16_stages on the shared and the per-sample route (bf16)
  cfg1_<prec>       the class-conditional MNIST model, fp32 and bf16
  tap_<part>        cfg2 at 64x64 on the shared route with layer1.<part> armed: that 128-wide layer leaves its fused kernel
  x_off, out_off    x or out starting 4 bytes into its storage: the scalar patch_in / patch_out kernels

Recording: `python tests/test_gpu_engine_routes.py OUT.json [CASE ...]` runs the named cases (default: those the golden file lacks) on
the GPU and writes the golden file with them to OUT.json.
"""
import json
import sys

import pytest
import torch

from conftest import GOLDEN
from test_gpu_bf16_stages import CONFIGS, ROUTES, latent, make

DEV = "cuda"
CASES = ([f"{c}/{r}" for c in dict(ROUTES) for r in ("shared", "per_sample")] + ["cfg1_fp32", "cfg1_bf16"] +
         [f"tap_{p}" for p in ("qkv", "ao", "geglu")] + ["x_off", "out_off"])


def _offset(t):
    """a contiguous copy of t whose data starts 4 bytes into its storage"""
    v = torch.empty(t.numel() + 1, device=t.device, dtype=t.dtype)[1:].view_as(t)
    v.copy_(t)
    return v


def route_families(case):
    """-> the launch families of one Engine.forward for this case, in launch order"""
    from k_diffusion import _native as N_
    from test_gpu_parity import build
    prec, tap, out = N_.PREC_BF16, None, None
    if case.startswith("cfg1_"):
        cfg, _, inner, _, z = build("cfg1_mnist", precision=case[5:])
        prec = inner.resolved_precision()
        eng = inner.engine()
        img, s_d, sd_ = z["x"][:2].to(DEV), z["sigma"][:2].to(DEV), cfg["model"]["sigma_data"]
        table, stride = eng.conditioning(s_d, class_cond=z["class_cond"][:2].to(DEV)), eng.cond_stride
    else:
        config, route = case.split("/") if "/" in case else ("cfg2_64_b3", "shared")
        raw_fn, H, W, sigmas, _ = CONFIGS[config]
        inner, P = make(raw_fn(), H, W)
        eng = inner.to(DEV).eval().engine()
        sigma = torch.tensor(sigmas)
        img, s_d, sd_ = latent(7, len(sigmas), H, W, sigma).to(DEV), sigma.to(DEV), P.sigma_data
        shared = route == "shared"
        table, stride = eng.conditioning(s_d[:1] if shared else s_d), 0 if shared else eng.cond_stride
        if case.startswith("tap_"):
            L = P.layers[1]
            tap = (f"layer1.{case[4:]}", len(sigmas) * (H // 4) * (W // 4) * {"qkv": 3 * L.C, "ao": L.C, "geglu": L.F}[case[4:]])
        elif case == "x_off":
            img = _offset(img)
        elif case == "out_off":
            out = _offset(torch.empty_like(img))
    eng.forward(img, s_d, table, stride, sd_, prec, out=out)         # first forward on this grid builds the position tables
    if tap is not None:
        eng.arm_tap(*tap, DEV)
    torch.cuda.synchronize()
    with N_.profile() as p:
        eng.forward(img, s_d, table, stride, sd_, prec, out=out)
    torch.cuda.synchronize()
    if tap is not None:
        assert eng.tap_count() == tap[1], f"tap {tap[0]}: {eng.tap_count()} elements, expected {tap[1]}"
    return [f for f, _ in p.launches]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_engine_route(case):
    want = json.loads((GOLDEN / "engine_routes.json").read_text())[case]
    got = route_families(case)
    assert got == want, f"{case}: launches\n  {got}\nexpected\n  {want}"


# the benchmark's neighbourhood models: every attention layer runs on a tensor-core kernel (attn_na_kernel at the two neighbourhood
# levels, attn_ws_kernel at the global level), none on attn_generic
BENCH_NA = {"cfg3_256_b2": "cfg3", "cfg5_512_b2": "cfg5"}


@pytest.mark.parametrize("case", [f"{c}/{r}" for c in BENCH_NA for r in ("shared", "per_sample")])
def test_benchmark_na_models_route_every_attention_to_tensor_cores(case):
    from test_gpu_bf16_stages import bench_raw
    routes = json.loads((GOLDEN / "engine_routes.json").read_text())
    assert case in routes, f"{case} is not recorded"
    depths = bench_raw(BENCH_NA[case.split("/")[0]])["model"]["depths"]
    n_attn = 2 * sum(depths[:-1]) + depths[-1]            # down and up layers of every outer level, then the middle level
    seq = routes[case]
    assert "attn_generic" not in seq
    assert seq.count("attn_tc") == n_attn, f"{seq.count('attn_tc')} attn_tc launches, {n_attn} attention layers"


if __name__ == "__main__":
    golden = json.loads((GOLDEN / "engine_routes.json").read_text())
    todo = sys.argv[2:] or [c for c in CASES if c not in golden]
    for c in todo:
        golden[c] = route_families(c)
        print(c, len(golden[c]), "launches")
    ordered = {c: golden[c] for c in CASES if c in golden}
    with open(sys.argv[1], "w") as f:
        f.write(json.dumps(ordered, indent=1) + "\n")
