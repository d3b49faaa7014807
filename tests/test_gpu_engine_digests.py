"""The exact fp32 engines bit for bit: SHA-256 digests of the U-Net denoiser of the four reference configs (with and without aug_cond),
every U-Net tap of mnist, the conditioning tables of both model families, and the transformer's fp32 forward, forward-mode (JVP) and
reverse-mode (VJP) outputs on cfg1 and the cfg2 model at 64x64, against tests/golden/engine_digests.json.  The other GPU tests compare
these paths with an oracle to a tolerance; these digests pin every bit, so a change of accumulation order in any kernel of the fp32
paths shows here.  The engine's workspace is filled with NaN before each call, so a read of a buffer no launch wrote changes a digest.

Record the golden (on the build whose results are the reference):  python tests/test_gpu_engine_digests.py --record OUT.json
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
GOLDEN = ROOT / "tests" / "golden" / "engine_digests.json"
DEV = "cuda"
UNETS = ["32x32_small", "32x32_small_butterflies", "cifar10", "mnist"]
TRANSFORMERS = ["cfg1_mnist", "sw64"]


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _nan_workspace(eng, need):
    """the engine's workspace of `need` bytes, every whole float of it NaN"""
    ws = eng._reserve(need, torch.device(DEV))
    n = ws.numel()
    ws[: n - n % 4].view(torch.float32).fill_(float("nan"))


def unet_digests(name):
    from conftest import load_npz
    from k_diffusion import _native
    from oracle.unet_oracle import stage_plan
    from test_gpu_unet import build
    cfg, _, model, den = build(name)
    eng = model.engine()
    z = load_npz(f"unet_{name}.npz")
    x, sig, aug = z["x"].to(DEV), z["sigma"].to(DEV), z["aug_cond"].to(DEV)
    B, _, H, W = x.shape
    need = int(_native.lib().kdb_unet_workspace_bytes(eng._h, _native.PREC_FP32, B, H, W))
    rec = {}
    for key, kw in (("denoised", {}), ("denoised aug", {"aug_cond": aug})):
        _nan_workspace(eng, need)
        rec[key] = _digest(den(x, sig, **kw))
    if name != "mnist":
        return rec
    rec["cond"] = _digest(eng.conditioning(sig))
    rec["cond aug"] = _digest(eng.conditioning(sig, aug))
    cond = eng.conditioning(sig, aug)
    for tap in ["patch_in", *stage_plan(cfg["model"])]:
        _nan_workspace(eng, need)
        buf = eng.arm_tap(tap, 1 << 24, x.device)
        eng.forward(x, sig, cond, eng.cond_stride, 0.0, _native.PREC_FP32)
        n = eng.tap_count()
        assert n > 0, tap
        rec[f"tap {tap}"] = _digest(buf[:n])
    return rec


def transformer_digests(stem):
    from k_diffusion import _native
    from test_gpu_parity import build
    cfg, _, inner, _, _ = build(stem)
    mcfg = cfg["model"]
    C, (H, W), sd = mcfg["input_channels"], mcfg["input_size"], float(mcfg["sigma_data"])
    B = 3
    g = torch.Generator().manual_seed(17)
    x = (torch.randn(B, C, H, W, generator=g) * 2).to(DEV)
    v = torch.randn(B, C, H, W, generator=g).to(DEV)
    u = torch.randn(B, C, H, W, generator=g).to(DEV)
    aug = (torch.randn(B, 9, generator=g) * 0.5).to(DEV)
    sig = torch.tensor([0.05, 1.3, 20.0], device=DEV)
    kw = {"class_cond": torch.tensor([1, 9, 4], device=DEV)} if inner.class_emb is not None else {}
    eng = inner.engine()
    cond = inner.conditioning(sig, aug, **kw)
    L, P = _native.lib(), _native.PREC_FP32
    rec = {"cond aug": _digest(cond)}
    _nan_workspace(eng, L.kdb_model_workspace_bytes(eng._h, P, B, H, W))
    rec["forward"] = _digest(eng.forward(x, sig, cond, eng.cond_stride, sd, P))
    _nan_workspace(eng, L.kdb_model_workspace_bytes(eng._h, P, 2 * B, H, W))
    out, tangent = eng.forward_jvp(x, v, sig, cond, eng.cond_stride, sd)
    rec["jvp out"], rec["jvp tangent"] = _digest(out), _digest(tangent)
    _nan_workspace(eng, L.kdb_model_vjp_workspace_bytes(eng._h, B, H, W))
    out, grad = eng.forward_vjp(x, u, sig, cond, eng.cond_stride, sd)
    rec["vjp out"], rec["vjp grad"] = _digest(out), _digest(grad)
    return rec


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("name", UNETS)
def test_unet_digests(golden, name):
    assert unet_digests(name) == golden[f"unet {name}"]


@pytest.mark.gpu
@pytest.mark.parametrize("stem", TRANSFORMERS)
def test_transformer_fp32_digests(golden, stem):
    assert transformer_digests(stem) == golden[f"transformer {stem}"]


if __name__ == "__main__":
    assert len(sys.argv) == 3 and sys.argv[1] == "--record", __doc__
    rec = {f"unet {n}": unet_digests(n) for n in UNETS}
    rec.update({f"transformer {s}": transformer_digests(s) for s in TRANSFORMERS})
    Path(sys.argv[2]).write_text(json.dumps(rec, indent=1) + "\n")
    print(f"recorded {sum(len(v) for v in rec.values())} digests -> {sys.argv[2]}")
