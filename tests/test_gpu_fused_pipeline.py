"""The fused level-0 kernels (csrc/tc_ffn_fused.cuh, csrc/tc_attn_block.cuh) bit for bit: SHA-256 digests of the updated x and of the row
statistics against tests/golden/fused_level0_digests.json.  The schedule of the MMAs inside these kernels is free to change, the
arithmetic is not: every accumulator sees the same wgmma shapes in the same K order and every epilogue the same operations, so any
change of a digest is a change of the results.  The cases cover the ways work falls on CTAs and warpgroups: one tile or window per CTA,
an odd number of windows (the second warpgroup idles on the last tile), fewer tiles than SMs, an uneven number of tiles per CTA, both
shifts, and the level-0 shapes of the 256x256 model at batch 32.  ss_out starts as NaN, so a row whose statistic is not written
changes the digest (and fails the finiteness check).

Record the golden (on the build whose results are the reference):  python tests/test_gpu_fused_pipeline.py --record OUT.json
"""
import hashlib
import json
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
for p in (str(ROOT), str(ROOT / "k-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
GOLDEN = ROOT / "tests" / "golden" / "fused_level0_digests.json"
C = 128

# (M, d_ff, statistics written)
FFN_CASES = [
    (128, 192, True),                        # one tile: one CTA, the fewest chunks (3)
    (100 * 128, 384, True),                  # fewer tiles than SMs, one tile per CTA
    (100 * 128, 384, False),                 # ... without the output statistics
    ((132 * 2 + 5) * 128, 384, True),        # uneven tiles per CTA
    (1280, 512, True),                       # 8 chunks
    (32 * 64 * 64, 384, True),               # level 0 of the 256x256 model at batch 32
]
# (B, h, w, shift)
ATTN_CASES = [
    (1, 8, 8, 0), (1, 8, 8, 4),              # one window: one CTA, its second warpgroup idles
    (3, 8, 8, 4),                            # odd number of windows
    (1, 24, 16, 4), (3, 16, 40, 0),          # fewer tiles than SMs (3, 15), one tile per CTA
    (5, 64, 64, 0), (5, 64, 64, 4),          # 160 tiles: uneven tiles per CTA
    (32, 64, 64, 0), (32, 64, 64, 4),        # level 0 of the 256x256 model at batch 32
]


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _x(M, seed):
    """bf16 rows of varied magnitude and their sum(x^2) in slot 0 of [M, 8] (the other slots NaN: they must never be read); inputs are
    drawn on the CPU so that they are the same on every machine"""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, C, generator=g) * (0.5 + torch.rand(M, 1, generator=g) * 3)).to(torch.bfloat16)
    ss = torch.full((M, 8), float("nan"))
    ss[:, 0] = x.double().pow(2).sum(1).float()
    return x, ss


def run_ffn(M, F, with_ss):
    from k_diffusion import _native as N_
    x, ss = _x(M, M + F)
    g = torch.Generator().manual_seed(7 * F + 1)
    w_up = (torch.randn(2 * F, C, generator=g) / C ** 0.5).to(torch.bfloat16)
    w_dn = (torch.randn(C, F, generator=g) / F ** 0.5).to(torch.bfloat16)
    ss_out = torch.full((M, 8), float("nan"), device="cuda") if with_ss else None
    got = N_.ffn_fused_bf16(x.cuda(), w_up.cuda(), w_dn.cuda(), ss.cuda(), ss_out)
    torch.cuda.synchronize()
    return got, ss_out


def run_attn(B, h, w, shift):
    from k_diffusion import _native as N_
    from oracle import kdiff_oracle as O
    M = B * h * w
    x, ss = _x(M, B * 1000 + h * 10 + w + shift)
    g = torch.Generator().manual_seed(h + w + shift)
    w_qkv = (torch.randn(3 * C, C, generator=g) / C ** 0.5).to(torch.bfloat16)
    w_out = (torch.randn(C, C, generator=g) / C ** 0.5).to(torch.bfloat16)
    theta = O.rope_theta(O.make_axial_pos(h, w), O.rope_freqs(64, 2))
    ss_out = torch.full((M, 8), float("nan"), device="cuda")
    got = N_.attn_block_bf16(x.view(B, h, w, C).cuda(), w_qkv.cuda(), w_out.cuda(), theta.cuda(), torch.tensor([10.0, 6.5], device="cuda"), shift,
                             ss.cuda(), ss_out)
    torch.cuda.synchronize()
    return got, ss_out


def _ffn_key(M, F, with_ss):
    return f"ffn M{M} F{F}" + ("" if with_ss else " no-ss")


def _attn_key(B, h, w, shift):
    return f"attn B{B} {h}x{w} shift{shift}"


def _digests(got, ss_out):
    d = {"x": _digest(got)}
    if ss_out is not None:
        d["ss"] = _digest(ss_out)
    return d


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("M,F,with_ss", FFN_CASES)
def test_ffn_fused_digests(golden, M, F, with_ss):
    got, ss_out = run_ffn(M, F, with_ss)
    assert bool(torch.isfinite(got.float()).all())
    if ss_out is not None:
        assert bool(torch.isfinite(ss_out[:, 0]).all()), "a row statistic was not written"
        assert bool(torch.isnan(ss_out[:, 1:]).all())
    assert _digests(got, ss_out) == golden[_ffn_key(M, F, with_ss)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,h,w,shift", ATTN_CASES)
def test_attn_block_digests(golden, B, h, w, shift):
    got, ss_out = run_attn(B, h, w, shift)
    assert bool(torch.isfinite(got.float()).all())
    assert bool(torch.isfinite(ss_out[:, 0]).all()), "a row statistic was not written"
    assert bool(torch.isnan(ss_out[:, 1:]).all())
    assert _digests(got, ss_out) == golden[_attn_key(B, h, w, shift)]


if __name__ == "__main__":
    assert len(sys.argv) == 3 and sys.argv[1] == "--record", __doc__
    rec = {_ffn_key(*c): _digests(*run_ffn(*c)) for c in FFN_CASES}
    rec.update({_attn_key(*c): _digests(*run_attn(*c)) for c in ATTN_CASES})
    Path(sys.argv[2]).write_text(json.dumps(rec, indent=1) + "\n")
    print(f"recorded {len(rec)} digests -> {sys.argv[2]}")
