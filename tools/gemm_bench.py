#!/usr/bin/env python
"""Device time of every generic token-stream GEMM launch (gemm_wg_kernel: level-1 and middle-level projections, merges, splits) of
one denoiser evaluation, each with the epilogue the model runs it with, against its hardware bound.  Run on the GPU box:

    python tools/gemm_bench.py [--configs cfg2 cfg5] [--repeat 20] [--json out.json]

The library is the one k_diffusion._native loads: $KDB200_LIB if set, so two builds can be compared by alternating calls.  Each
evaluation is enqueued behind a gate kernel (kernels back to back, as in a graph replay) with CUDA events around every launch; a
launch's time is the median over --repeat evaluations.  Bound = max(FLOPs / 989 TFLOP/s, minimum bytes / 3.35 TB/s), the H100 SXM
data-sheet figures (dense BF16, HBM3); minimum bytes = A + W + output, plus the residual / skip tensor of out / down / split.

Operand stream = the A and W bytes the CTAs' TMA rings load from L2, from the tile shapes (every 128 x BN tile loads one A and one W
k-block per 64-wide k-step), and the same over the launch's time in TB/s.  No L2 bandwidth is printed against it: none has been
measured for this access pattern.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch

import k_diffusion as K
from k_diffusion import _native

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
CONFIGS = {
    # cfg2: the benchmark's headline model (256 x 256, widths 128 / 256 / 512), batch 32
    "cfg2": (lambda: json.loads((ROOT / "tests/golden/cfg2_sw256_shapes.json").read_text())["config"], 32),
    # cfg5: 512 x 512, widths 256 / 512 / 1024, batch 16
    "cfg5": (lambda: {"model": {"type": "image_transformer_v2", "input_channels": 3, "input_size": [512, 512], "patch_size": [4, 4],
                                "depths": [2, 2, 4], "widths": [256, 512, 1024], "sigma_data": 0.5, "sigma_min": 1e-2, "sigma_max": 160}}, 16),
}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), (s.strip() for s in out.splitlines()[0].split(","))))
    except (OSError, subprocess.CalledProcessError):
        return {"name": torch.cuda.get_device_name()}


def min_bytes(label, M, N, K):
    out = M * N // 2 if "geglu" in label else M * N
    extra = M * N if ("res" in label or label.startswith("split")) else 0
    return 2 * (M * K + N * K + out + extra)


def operand_bytes(M, N, K):
    """A + W bytes the GEMM's rings load: 128 x BN tiles (BN = 128, or 64 when N % 128 != 0), a 128 x 64 A and a BN x 64 W k-block each"""
    bn = 128 if N % 128 == 0 else 64
    return -(-M // 128) * (N // bn) * (K // 64) * (128 + bn) * 64 * 2


def bench(name, repeat):
    raw, batch = CONFIGS[name]
    cfg = K.config.load_config(raw())
    res = cfg["model"]["input_size"][0]
    inner = K.synth.synth_init_(K.config.make_model(cfg), seed=1).cuda().eval().set_precision("bf16")
    x = torch.randn(batch, 3, res, res, device="cuda") * 10
    sig = torch.full([batch], 3.0, device="cuda")
    eng = inner.engine()
    table = eng.conditioning(sig[:1])

    def evaluate():
        return eng.forward(x, sig, table[0], 0, float(cfg["model"]["sigma_data"]), inner.resolved_precision())

    for _ in range(3):
        evaluate()
    torch.cuda.synchronize()
    seq = K.models.flops.launch_layers(cfg["model"], batch)
    times = [[] for _ in seq]
    for _ in range(repeat):
        with _native.profile(gate_ms=20.0) as prof:
            evaluate()
        gemms = [ms for fam, ms in prof.launches if fam.startswith("gemm")]
        assert len(gemms) == len(seq), f"{len(gemms)} GEMM-family launches, {len(seq)} expected"
        for i, ms in enumerate(gemms):
            times[i].append(ms)
    rows = []
    for (label, M, N, Kd, macs), ts in zip(seq, times):
        if "fused" in label:
            continue
        us = sorted(ts)[len(ts) // 2] * 1e3
        flop, byts = 2.0 * macs, min_bytes(label, M, N, Kd)
        t_mma, t_hbm = flop / (PEAK_TFLOPS * 1e12) * 1e6, byts / (PEAK_TBS * 1e12) * 1e6
        opnd = operand_bytes(M, N, Kd)
        rows.append(dict(label=label, M=M, N=N, K=Kd, us=round(us, 2), tflops=round(flop / us / 1e6, 1), gbs=round(byts / us / 1e3),
                         bound_us=round(max(t_mma, t_hbm), 2), bound_by="MMA" if t_mma >= t_hbm else "HBM",
                         operand_mb=round(opnd / 1e6, 1), operand_tbs=round(opnd / us / 1e6, 2)))
    return dict(config=name, batch=batch, generic_gemm_us=round(sum(r["us"] for r in rows), 1),
                bound_us=round(sum(r["bound_us"] for r in rows), 1), operand_mb=round(sum(r["operand_mb"] for r in rows), 1), launches=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["cfg2", "cfg5"], choices=sorted(CONFIGS))
    ap.add_argument("--repeat", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_bench measures on the GPU"
    res = dict(gpu=gpu_info(), lib=str(_native.LIB_PATH), configs=[bench(c, a.repeat) for c in a.configs])
    print(json.dumps(res["gpu"]), res["lib"])
    for c in res["configs"]:
        print(f"{c['config']} B={c['batch']}: generic GEMMs {c['generic_gemm_us']:.1f} us per evaluation (bound {c['bound_us']:.1f} us); "
              f"operand stream {c['operand_mb']:.0f} MB")
        for r in c["launches"]:
            print(f"  {r['label']:16s} {r['M']:6d} x {r['N']:5d} x {r['K']:5d}  {r['us']:8.2f} us  {r['tflops']:6.1f} TFLOP/s  "
                  f"{r['gbs']:5d} GB/s  bound {r['bound_us']:6.2f} us ({r['bound_by']}, {r['bound_us'] / r['us']:5.1%})  "
                  f"operands {r['operand_mb']:6.1f} MB {r['operand_tbs']:5.2f} TB/s")
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
