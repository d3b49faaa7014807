"""The tensor-core neighbourhood attention kernel (attn_na_kernel: kdb_attention's bf16 fast path for 7x7 neighbourhoods) value by
value against a float64 reference over gathered keys.

Reference.  Query (i, j) sees the NATTEN window, rows [clamp(i - 3, 0, h - 7), +7) x columns [clamp(j - 3, 0, w - 7), +7): always 49
keys, shifted inward at the borders.  na_keys builds that [T, 49] key-index table, so the reference costs O(T 49) and runs at 128 x 128
tokens and batch 16 (with plain torch ops, in float64, on the device of its inputs).  P is rounded where the kernel rounds it
(tc_attention.cu, pass B):
    p = bf16(exp(s - shift)),  l = the sum of those bf16 values,  out = (p v) / l,
    shift = the logit bound when one is given (one pass), else the row maximum over the 49 keys (pass A).
The kernel computes s, the exponent, l and P V in fp32 and stores out as bf16.

Tolerance, per element, for the reference output y:
    |got - y| <= halfulp(y) + 2 (flip + 2^-14 sum_i p_i |v_i| / l)
* halfulp(y), half a bf16 ulp at y: the output store.  For any x, |bf16(x) - y| <= halfulp(y) + 2 |x - y| (a rounding that crosses
  into the next binade at most doubles |x - y|), so the other terms bound |x - y| for the kernel's fp32 result x.
* flip: before its rounding the kernel's p differs from exp(s - shift) by the fp32 logit (64 exact products summed in fp32:
  <= 64 2^-24 |q| |k| <= 1.5e-4 at the largest bound, 40), the exponent's fma and exp2f (~1e-5).  That is below DELTA = 2^-11 of
  p, so p_i can round to the other neighbour than the reference's only where exp(s_i - shift) lies within DELTA p_i of a bf16
  midpoint.  Such a key moves out by ulp(p_i) |v_i - y| / l; flip sums that over the keys of the row that are this close.
* 2^-14 sum p |v| / l: fp32 sums of at most 128 terms for l and P V (128 2^-24 = 2^-17, with 8x to spare).
test_gpu_attn_persistent.py's band, 8e-3 |y| + 8e-3 elementwise and 2.5e-3 mean |y| on average, is several times wider.  It
accepts a kernel that rounds P for P V but sums l from the unrounded p, which changes l coherently by up to U = 2^-8.  The bound
above rejects that.  Every GPU case asserts both the bound above and the persistent test's band.

The CPU leg runs without a GPU.  It shows that the gathered reference equals the oracle's dense masked attention, that the
tolerance accepts an emulation of the kernel's fp32 arithmetic, and that it rejects each near miss a kernel could make:
  noclamp      the window centred on the query and cut at the border instead of shifted inward
  row_off      the window one row lower;  col_off  one column to the right
  halo_row     the last row of the query block's 14 x 22 key halo dropped (the third 5/5/4-row key box one row short)
  head         the next head's keys
  l_unrounded  l summed from p before its rounding to bf16
"""
import math

import pytest
import torch

DEV = "cuda"
KS = 7                  # neighbourhood size: the kernel is built for 7 x 7
QH, KH = 8, 14          # the kernel's query block height and its key halo height
SCALE = 10.0            # cosine-similarity scale of the test data: |q . k| <= SCALE
MAX_BOUND = 40.0        # KDB_ATTN_MAX_BOUND (tc_kernels.cuh): the largest logit bound the engine hands the kernels
LOG2E = 1.4426950408889634
DELTA = 2.0 ** -11      # relative error of the kernel's p before its bf16 rounding is below this (docstring)
NEAR_MISSES = ("noclamp", "row_off", "col_off", "halo_row", "head", "l_unrounded")


def bf(t):
    return t.to(torch.bfloat16).to(t.dtype)


def na_keys(h, w, nm=None, device="cpu"):
    """-> (idx [h w, 49] key token of each query's window, ok [h w, 49] whether that key is attended)"""
    i, j = torch.arange(h, device=device), torch.arange(w, device=device)
    rs, cs = (i - KS // 2).clamp(0, h - KS), (j - KS // 2).clamp(0, w - KS)
    if nm == "noclamp":
        rs, cs = i - KS // 2, j - KS // 2
    elif nm == "row_off":
        rs = (i - KS // 2 + 1).clamp(0, h - KS)
    elif nm == "col_off":
        cs = (j - KS // 2 + 1).clamp(0, w - KS)
    d = torch.arange(KS, device=device)
    kr = (rs[:, None] + d).view(h, 1, KS, 1).expand(h, w, KS, KS)
    kc = (cs[:, None] + d).view(1, w, 1, KS).expand(h, w, KS, KS)
    ok = (kr >= 0) & (kr < h) & (kc >= 0) & (kc < w)
    if nm == "halo_row":
        r0 = ((i // QH) * QH - KS // 2).clamp(0, h - KH)          # the query block's halo origin (tc_attention.cu r0)
        ok = ok & (kr != (r0 + KH - 1).view(h, 1, 1, 1))
    idx = kr.clamp(0, h - 1) * w + kc.clamp(0, w - 1)
    return idx.reshape(h * w, KS * KS), ok.reshape(h * w, KS * KS)


def na_logits(q, k, nm=None):
    """q, k [B, h, w, nh, e] -> (s [B, h w, nh, 49] with -inf outside the window, idx, ok)"""
    B, h, w, nh, e = q.shape
    idx, ok = na_keys(h, w, nm, q.device)
    qf, kf = q.reshape(B, h * w, nh, e), k.reshape(B, h * w, nh, e)
    if nm == "head":
        kf = kf.roll(-1, 2)
    s = torch.stack([(qf * kf[:, idx[:, o]]).sum(-1) for o in range(KS * KS)], -1)
    return s.masked_fill(~ok[:, None, :], float("-inf")), idx, ok


def halfulp(y):
    """half the spacing of bf16 values at y (8-bit significand)"""
    _, E = torch.frexp(y)
    return torch.where(y == 0, torch.zeros_like(y), torch.ldexp(torch.ones_like(y), E - 9))


def na_attention(q, k, v, bound=None, *, kernel=False, p_bf16=True, nm=None, with_tol=False):
    """7x7 neighbourhood attention (scale 1) of q, k, v [B, h, w, nh, e], computed in their dtype -> [B, h, w, nh, e].

    bound [nh] or None: the softmax shift (None: the row maximum).  p_bf16: round p to bf16 for P V and l.  kernel: the kernel's
    formula exp2(s log2e - shift log2e) and its bf16 output store (give fp32 inputs to emulate its arithmetic).  nm: a near miss.
    with_tol: -> (out, tolerance of a kernel's output against out; see the module docstring)."""
    B, h, w, nh, e = q.shape
    s, idx, ok = na_logits(q, k, nm)
    vf = v.reshape(B, h * w, nh, e)
    shift = s.amax(-1, keepdim=True) if bound is None else bound.to(s).view(nh, 1)
    p = torch.exp2(s * LOG2E - shift * LOG2E) if kernel else torch.exp(s - shift)
    pr = bf(p) if p_bf16 else p
    l = (p if nm == "l_unrounded" else pr).sum(-1, keepdim=True)
    o = sum(pr[..., i, None] * vf[:, idx[:, i]] for i in range(KS * KS))
    y = bf(o * (1 / l)) if kernel else o / l
    out = y.reshape(B, h, w, nh, e)
    if not with_tol:
        return out
    _, E = torch.frexp(p)
    ulp = torch.ldexp(torch.ones_like(p), E - 8)
    frac = p / ulp
    near = (p > 0) & (((frac - frac.floor()) - 0.5).abs() * ulp <= DELTA * p)
    wflip = torch.where(near, ulp, torch.zeros_like(p))
    flip = sum(wflip[..., i, None] * (vf[:, idx[:, i]] - y).abs() for i in range(KS * KS)) / l
    spread = sum(pr[..., i, None] * vf[:, idx[:, i]].abs() for i in range(KS * KS)) / l
    tol = halfulp(y) + 2 * (flip + 2.0 ** -14 * spread)
    return out, tol.reshape(B, h, w, nh, e)


def make_qkv(B, h, w, nh, seed, scale=SCALE, region=None, device=DEV):
    """qkv [B, h*w, 3*nh*64] bf16 with cosine-normalised q, k (|q| = |k| = sqrt(scale)), as test_gpu_attn_persistent._qkv.

    region (r0, r1, c0, c1, kind) overwrites the tokens of rows [r0, r1) x columns [c0, c1):
      "opposed"   q ~ u and k ~ -u (one direction u per head): every logit of a query inside is near -scale
      "two_keys"  k alternates between two vectors by column: each row's p takes two values, both rounded in the bounded softmax and
                  the smaller one in the row-maximum softmax (the rows where l summed from unrounded p shows)"""
    g = torch.Generator(device=device).manual_seed(seed)
    t = torch.randn(B, h, w, 3, nh, 64, device=device, generator=g)
    if region is not None:
        r0, r1, c0, c1, kind = region
        n = (r1 - r0, c1 - c0, nh, 64)
        if kind == "opposed":
            u = torch.randn(nh, 64, device=device, generator=g)
            t[:, r0:r1, c0:c1, 0] = u + 0.02 * torch.randn(B, *n, device=device, generator=g)
            t[:, r0:r1, c0:c1, 1] = -u - 0.02 * torch.randn(B, *n, device=device, generator=g)
        else:
            kk = torch.randn(2, nh, 64, device=device, generator=g)
            t[:, r0:r1, c0:c1, 1] = kk[torch.arange(c0, c1, device=device) % 2]
    t[..., :2, :, :] = t[..., :2, :, :] / t[..., :2, :, :].norm(dim=-1, keepdim=True) * scale ** 0.5
    return t.to(torch.bfloat16).reshape(B, h * w, 3 * nh * 64).contiguous()


def split(qkv, h, w, nh, dtype):
    B = qkv.shape[0]
    return qkv.to(dtype).view(B, h, w, 3, nh, 64).unbind(3)


def check(got, want, tol, what):
    """-> list of failures: the bound of the docstring, the persistent test's band and its mean bound"""
    err = (got.double() - want).abs()
    bad = []
    if not bool((err <= tol).all()):
        r = err / tol
        i = int(r.argmax())
        bad.append(f"{what}: {int((r > 1).sum())} elements out of tolerance, max err/tol {float(r.flatten()[i]):.3g} "
                   f"(err {float(err.flatten()[i]):.3g}, want {float(want.flatten()[i]):.4g})")
    if not bool((err <= 8e-3 * want.abs() + 8e-3).all()):
        bad.append(f"{what}: outside 8e-3 |y| + 8e-3, max err {float(err.max()):.3g}")
    if not float(err.mean()) < 2.5e-3 * float(want.abs().mean()):
        bad.append(f"{what}: mean err {float(err.mean()):.3g} >= 2.5e-3 mean |y|")
    return bad


def max_ratio(got, want, tol):
    return float(((got.double() - want).abs() / tol).max())


# ----------------------------------------------------------------------------------------------------------------------------
# GPU: the kernel
# ----------------------------------------------------------------------------------------------------------------------------
def _run(qkv, h, w, nh, bound):
    from k_diffusion import _native as N_
    B = qkv.shape[0]
    out = torch.full((B, h * w, nh * 64), float("nan"), dtype=torch.bfloat16, device=DEV)
    N_.check(N_.lib().kdb_attention(N_.PREC_BF16, 1, N_.ptr(qkv), N_.ptr(out), B, h, w, nh, 64, N_._ATTN_CODE["neighborhood"], KS, 0,
                                    N_.ptr(bound), N_.stream()))
    torch.cuda.synchronize()
    return out


def _check_kernel(qkv, h, w, nh, bound):
    from k_diffusion import _native as N_
    B = qkv.shape[0]
    before = N_.launch_breakdown().get("attn_tc", 0)
    got = _run(qkv, h, w, nh, bound)
    # the tensor-core kernel ran: a shape that fell back to the generic kernel would pass the value checks for the wrong reason
    assert N_.launch_breakdown().get("attn_tc", 0) == before + 1, "attn_na_kernel did not run"
    assert not bool(torch.isnan(got).any()), "an output element was not written"
    want, tol = na_attention(*split(qkv, h, w, nh, torch.float64), bound, with_tol=True)
    bad = check(got.view(want.shape), want, tol, "kernel")
    print(f"B={B} {h}x{w} nh={nh} {'bounded' if bound is not None else 'row-max'}: max err/tol {max_ratio(got.view(want.shape), want, tol):.3f}")
    assert not bad, "\n".join(bad)
    again = _run(qkv, h, w, nh, bound)
    assert torch.equal(got.view(torch.int16), again.view(torch.int16)), "two runs differ"
    alone = _run(qkv[B - 1:].contiguous(), h, w, nh, bound)
    assert torch.equal(got[B - 1:].view(torch.int16), alone.view(torch.int16)), "an image alone differs from the same image in the batch"
    return want


CASES = [
    # B, h, w, nh
    (2, 16, 32, 2),         # the smallest grid the kernel takes: both query blocks of a column clamp their halo on both axes
    (1, 24, 48, 1),         # an interior block on each axis (halo origin qi0 - 3, qj0 - 3), one head
    (2, 40, 64, 3),         # 5 row blocks (odd), odd head count
    (1, 16, 112, 2),        # wide: 7 column blocks
    (1, 120, 32, 1),        # tall: 15 row blocks (odd)
    (64, 64, 64, 2),        # cfg3 / cfg4 level 0 (256x256 model) at cfg3's batch
    (64, 32, 32, 4),        # cfg3 / cfg4 level 1
    (16, 128, 128, 4),      # cfg5 level 0 (512x512 model) at its batch
    (16, 64, 64, 8),        # cfg5 level 1
]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("bounded", [True, False], ids=["bounded", "row-max"])
@pytest.mark.parametrize("B,h,w,nh", CASES)
def test_attention_na_vs_reference(B, h, w, nh, bounded):
    qkv = make_qkv(B, h, w, nh, seed=B * 1000 + h * w + nh)
    _check_kernel(qkv, h, w, nh, torch.full([nh], SCALE, device=DEV) if bounded else None)


@pytest.mark.gpu
@pytest.mark.parametrize("bounded", [True, False], ids=["bounded", "row-max"])
def test_attention_na_at_the_largest_bound(bounded):
    """Scale and bound KDB_ATTN_MAX_BOUND (40), with a region where k ~ -q: every logit of the queries inside is near -40, so the
    bounded softmax's p = exp(s - 40) is near e^-80 (~1e-35: still a normal fp32 and bf16 number) and must stay accurate there."""
    B, h, w, nh = 2, 32, 48, 2
    region = (8, 24, 16, 40, "opposed")
    qkv = make_qkv(B, h, w, nh, seed=40, scale=MAX_BOUND, region=region)
    q, k, _ = split(qkv, h, w, nh, torch.float64)
    s = na_logits(q, k)[0].view(B, h, w, nh, KS * KS)
    inner = s[:, 11:21, 19:37]                       # queries whose whole window lies in the region
    assert float(inner.amax()) < -0.9 * MAX_BOUND, f"region logits reach {float(inner.amax()):.2f}"
    want = _check_kernel(qkv, h, w, nh, torch.full([nh], MAX_BOUND, device=DEV) if bounded else None)
    assert float(want[:, 11:21, 19:37].abs().mean()) > 0.05            # the region's outputs are not vanishing


# ----------------------------------------------------------------------------------------------------------------------------
# CPU leg
# ----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(7, 7), (9, 12), (16, 32), (24, 48), (13, 8)])
def test_gathered_reference_equals_dense_oracle(h, w):
    """With an unrounded softmax the gathered reference is the oracle's dense masked neighbourhood attention."""
    from oracle import kdiff_oracle as O
    q, k, v = split(make_qkv(2, h, w, 3, seed=h * w, device="cpu"), h, w, 3, torch.float64)
    want = O.neighborhood_attention(q, k, v, KS)
    got = na_attention(q, k, v, p_bf16=False)
    # both in float64; the bound leaves room for the CPU's vectorised exp and summation orders (up to ~1e-9 seen), far below the
    # > 1e-2 that a misplaced window moves outputs by
    assert float((got - want).abs().max()) < 1e-8


@pytest.mark.parametrize("bounded", [True, False], ids=["bounded", "row-max"])
@pytest.mark.parametrize("B,h,w,nh", [(1, 16, 32, 2), (1, 24, 48, 2)])
def test_tolerance_accepts_emulation_and_rejects_near_misses(B, h, w, nh, bounded):
    """The kernel's arithmetic emulated on the CPU (fp32 logits, exponent, l and P V; bf16 P and output) passes the bound and the
    persistent test's band; a kernel with each near miss puts at least one element outside the bound.  The grids have a
    bottom-clamped query block (16 x 32) and interior blocks (24 x 48); rows 4-12 hold the two-key region."""
    qkv = make_qkv(B, h, w, nh, seed=7 * h + w, region=(4, 12, 0, w, "two_keys"), device="cpu")
    bound = torch.full([nh], SCALE) if bounded else None
    want, tol = na_attention(*split(qkv, h, w, nh, torch.float64), bound, with_tol=True)
    q, k, v = split(qkv, h, w, nh, torch.float32)
    got = na_attention(q, k, v, bound, kernel=True)
    bad = check(got, want, tol, "emulation")
    print(f"emulation: max err/tol {max_ratio(got, want, tol):.3f}")
    assert not bad, "\n".join(bad)
    missed = []
    for nm in NEAR_MISSES:
        wrong = na_attention(q, k, v, bound, kernel=True, nm=nm)
        r = (wrong.double() - want).abs() / tol
        print(f"near miss {nm:>12s}: max err/tol {float(r.max()):.2f} ({int((r > 1).sum())} out)")
        if not bool((r > 1).any()):
            missed.append(f"near miss {nm} passes (max err/tol {float(r.max()):.3f})")
    assert not missed, "\n".join(missed)


def test_near_miss_windows_differ_where_expected():
    """The near-miss key tables change the windows they name and no others (so a rejection is the named mistake)."""
    h, w = 24, 48
    idx, ok = na_keys(h, w)
    assert bool(ok.all()) and bool((idx >= 0).all()) and int(idx.max()) < h * w
    assert idx.unique(dim=1).shape == idx.shape                      # 49 distinct keys per query
    qi = torch.arange(h * w) // w
    for nm, rows in (("row_off", (qi >= 3) & (qi < h - 4)), ("noclamp", None), ("col_off", None)):
        i2, ok2 = na_keys(h, w, nm)
        moved = ((i2 != idx) | ~ok2).any(1)
        if rows is not None:
            assert torch.equal(moved, rows), nm
        else:
            assert bool(moved.any()) and not bool(moved.all()), nm
    _, ok_h = na_keys(h, w, "halo_row")
    # the last halo row is in some window of every query block but the top one (whose halo is clamped to rows 0..13: windows end at row 10)
    dropped = (~ok_h).any(1).view(h, w).any(1)
    assert not bool(dropped[:QH].any()) and bool(dropped[QH:].any())
    assert math.isclose(float(halfulp(torch.tensor([1.0], dtype=torch.float64))), 2.0 ** -8)
