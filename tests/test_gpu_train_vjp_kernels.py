"""The transformer's reverse-mode kernels one by one on the H100 (kdb_gemm_vjp, kdb_rmsnorm_vjp, kdb_qknorm_rope_vjp, kdb_geglu_vjp,
kdb_split_vjp_gather, kdb_split_unpatch_lerp, kdb_merge_scatter_add, kdb_patch_out_vjp, kdb_patch_in_vjp, kdb_model_mapping_vjp): the
kernels kdb_model_forward_vjp / kdb_model_forward_train run between the loss and the parameter-gradient reductions, at the branches the
whole-model shapes never reach: ragged 64 x 64 tiles, several images per tile, M past the 65535-row-tile grid, accumulation into nonzero
gradients, per-image scale rows, every head width and both RoPE layouts, grid-stride loops, raw and Karras patch maps and the
patch_out shared-memory edge, and the mapping network at depth 1 to 8 with every conditioning input.

Exact operands (small integers) make every sum of products exact, so those kernels must equal the float64 sum bit for bit; the kernels that
move data or do one fp32 operation per element must equal the same torch expression on the GPU bit for bit.  Random operands hold each
element to an fp32 bound over float64 torch.func.vjp of the oracle's op.  Written outputs start as NaN and accumulated ones as nonzero
values, every output has a sentinel tail, and two calls give the same bits."""
import math

import pytest
import torch
from torch.nn import functional as F

from oracle import kdiff_oracle as O
from test_gpu_train import build
from test_gpu_train_kernels import SENTINEL, U, _assert_exact, _assert_written, _gen, _guarded, _ints

from k_diffusion import _native

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRID_STRIDE = 132 * 16 * 256      # elements in one pass of the elementwise kernels' grid (grid_stride_blocks)
ROW_CHUNK = 65535 * 64            # rows of one gemm_vjp launch


def _tail(n, pad=64):
    """(buffer, view): n floats to be filled by the caller followed by `pad` sentinel floats"""
    buf = torch.empty(n + pad, device=DEV)
    buf[n:] = SENTINEL
    return buf, buf[:n]


def _assert_bounded(got, want, bound, what=""):
    err = (got.double() - want).abs()
    ok = err <= bound
    assert ok.all(), (f"{what}: max error {err.max():.3e}, worst excess {(err - bound).max():.3e}, {int((~ok).sum())} elements out of "
                      f"bound, first at {(~ok).nonzero()[0].tolist()}")


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_gemm_vjp

# (M, N, K): one row, ragged M and K with N past one 16-wide step, the ada_total -> dcond product (M = B = 64, N = ada_total of the
# cifar10 transformer, 2 (4 x 256 + 4 x 256) + 4 (2 x 512), K = mw 256), config_mnist's qkv and down projections at B = 64 (3136 rows) and
# config_cifar10's at level 0 (16384 rows) and level 1 (4096 rows, d_ff 1536)
GEMM = [(1, 4, 4), (7, 12, 36), (9, 68, 132), (65, 100, 68), (64, 6144, 256), (3136, 768, 256), (3136, 256, 768), (16384, 768, 256),
        (4096, 512, 1536)]


def _run_gemm_vjp(dc, w):
    M, K = dc.shape[0], w.shape[1]
    buf, out = _guarded(M * K)
    got = _native.gemm_vjp(dc, w, out=out.view(M, K))
    _assert_written(buf, M * K)
    assert torch.equal(got, _native.gemm_vjp(dc, w)), "two calls differ"
    return got


@pytest.mark.parametrize("M,N,K", GEMM)
def test_gemm_vjp(M, N, K):
    g = _gen("gemm_vjp", M, N, K)
    dc, w = _ints((M, N), g), _ints((N, K), g)
    _assert_exact(_run_gemm_vjp(dc, w), dc.double().cpu() @ w.double().cpu())
    dc, w = torch.randn(M, N, device=DEV, generator=g), torch.randn(N, K, device=DEV, generator=g)
    a, b = dc.double(), w.double()
    _assert_bounded(_run_gemm_vjp(dc, w), a @ b, 1.01 * N * U * (a.abs() @ b.abs()), "dA")


@pytest.mark.parametrize("N,K", [(4, 4), (4, 8)])
def test_gemm_vjp_past_one_launch_of_rows(N, K):
    """M = 65535 * 64 + 65 rows: a second launch of 65 rows, one ragged tile of them; exact on integers.  With K != N the second launch's
    output offset (mo K) differs from its input offset (mo N)"""
    M = ROW_CHUNK + 65
    g = _gen("gemm_vjp_big", N, K)
    dc = torch.randint(-4, 5, (M, N), device=DEV, generator=g, dtype=torch.int8).float()
    w = _ints((N, K), g)
    got = _run_gemm_vjp(dc, w)
    _assert_exact(got, (dc.double() @ w.double()).cpu())
    del dc, got
    torch.cuda.empty_cache()


def _unpatch(d, hc, wc):
    """coarse rows [B hc wc, (nh nw e)] -> fine tokens [B, 2hc, 2wc, e] (the inverse of the TokenMerge gather)"""
    B, Cf = d.shape[0] // (hc * wc), d.shape[1] // 4
    return d.view(B, hc, wc, 2, 2, Cf).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * hc, 2 * wc, Cf)


def _run_unpatch_acc(dc, w, start, hc, wc):
    """kdb_gemm_vjp VJP_UNPATCH_ACC onto a copy of `start` with a sentinel tail, twice from the same start: -> result"""
    n = start.numel()
    buf, out = _tail(n)
    out.copy_(start.flatten())
    got = _native.gemm_vjp(dc, w, out=out.view(start.shape), unpatch=(hc, wc))
    assert (buf[n:] == SENTINEL).all(), "a write past the end of the fine tokens"
    again = start.clone()
    _native.gemm_vjp(dc, w, out=again, unpatch=(hc, wc))
    assert torch.equal(got, again), "two calls differ"
    return got


# (B, hc, wc, Cf, N): one token, several images per 64-row tile (15- and 6-token coarse grids, ragged K), 7 x 3 grids, and config_cifar10's
# merge at B = 64 (16 x 16 -> 8 x 8, 256 -> 512 channels)
UNPATCH = [(1, 1, 1, 1, 4), (9, 3, 5, 5, 12), (13, 2, 3, 17, 36), (5, 7, 3, 33, 68), (64, 8, 8, 256, 512)]


@pytest.mark.parametrize("B,hc,wc,Cf,N", UNPATCH)
def test_gemm_vjp_unpatch_accumulates(B, hc, wc, Cf, N):
    g = _gen("unpatch", B, hc, wc, Cf, N)
    M, K = B * hc * wc, 4 * Cf
    dc, w, start = _ints((M, N), g), _ints((N, K), g), _ints((B, 2 * hc, 2 * wc, Cf), g, -50, 50)
    got = _run_unpatch_acc(dc, w, start, hc, wc)
    _assert_exact(got, start.double().cpu() + _unpatch(dc.double().cpu() @ w.double().cpu(), hc, wc))
    dc, w = torch.randn(M, N, device=DEV, generator=g), torch.randn(N, K, device=DEV, generator=g)
    start = torch.randn(B, 2 * hc, 2 * wc, Cf, device=DEV, generator=g)
    a, b = dc.double(), w.double()
    want = start.double() + _unpatch(a @ b, hc, wc)
    _assert_bounded(_run_unpatch_acc(dc, w, start, hc, wc), want, 1.01 * (N + 1) * U * (start.double().abs() + _unpatch(a.abs() @ b.abs(), hc, wc)),
                    "dfine")


def test_gemm_vjp_unpatch_past_one_launch_of_rows():
    """1025 images of 64 x 64 coarse tokens: 4,198,400 rows, whole images per launch (1023 in the first, 2 in the second); exact"""
    B, hc, wc, Cf, N = 1025, 64, 64, 1, 4
    M = B * hc * wc
    assert M > ROW_CHUNK and ROW_CHUNK // (hc * wc) == 1023
    g = _gen("unpatch_big")
    dc = torch.randint(-4, 5, (M, N), device=DEV, generator=g, dtype=torch.int8).float()
    w = _ints((N, 4 * Cf), g)
    start = torch.randint(-50, 51, (B, 2 * hc, 2 * wc, Cf), device=DEV, generator=g, dtype=torch.int8).float()
    got = _run_unpatch_acc(dc, w, start, hc, wc)
    _assert_exact(got, (start.double() + _unpatch(dc.double() @ w.double(), hc, wc)).cpu())
    del dc, start, got
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_rmsnorm_vjp

def rmsnorm_bound(x, s, dy, C):
    """the fp32 roundings of dx += r (s dy) - x r^3 mean(x s dy): the row sums over C (and r's rsqrt) on the float64 magnitudes of both terms"""
    r = torch.rsqrt((x * x).mean(-1, keepdim=True) + 1e-6)
    t1 = r * (s * dy).abs()
    t2 = x.abs() * r ** 3 * (x * s * dy).abs().mean(-1, keepdim=True)
    return (2 * C + 24) * U * (t1 + t2)


# (rows, C, rows per image, per-image scale rows): one row, 7 and 9 rows (one CTA of 8 warps, and one more row), C 4, 33 and 96 (not
# multiples of 32), a shared scale row; config_mnist's AdaRMSNorm at B = 64 (3136 rows of 49 per image, the scale rows the conditioning
# table's, ada_total + mw apart) and config_cifar10's at level 0 and 1 (16384 x 256 and 4096 x 512)
RMS = [(1, 4, 1, False), (7, 33, 7, False), (9, 96, 3, True), (9, 4, 1, True), (50, 33, 10, True), (3136, 256, 49, True), (16384, 256, 256, True),
       (4096, 512, 64, True)]


@pytest.mark.parametrize("rows,C,R,per_image", RMS)
def test_rmsnorm_vjp_accumulates(rows, C, R, per_image):
    g = _gen("rmsnorm_vjp", rows, C, R)
    B = rows // R
    stride = C + 37 if per_image else 0
    x = torch.randn(rows, C, device=DEV, generator=g) * 2 + 0.5
    dy = torch.randn(rows, C, device=DEV, generator=g)
    scale = torch.randn((B - 1) * stride + C, device=DEV, generator=g) + 1
    dx0 = torch.randn(rows, C, device=DEV, generator=g)
    n = rows * C
    buf, out = _tail(n)
    out.copy_(dx0.flatten())
    got = _native.rmsnorm_vjp(x, dy, scale, out.view(rows, C), rows_per_image=R, scale_bstride=stride)
    assert (buf[n:] == SENTINEL).all(), "a write past the end of dx"
    again = _native.rmsnorm_vjp(x, dy, scale, dx0.clone(), rows_per_image=R, scale_bstride=stride)
    assert torch.equal(got, again), "two calls differ"
    rows_of = torch.arange(rows, device=DEV) // R
    s = torch.stack([scale[b * stride:b * stride + C] for b in range(B)]).double()[rows_of]
    x64, dy64 = x.double(), dy.double()
    _, pull = torch.func.vjp(lambda t: O.rms_norm(t, s), x64)
    want = dx0.double() + pull(dy64)[0]
    _assert_bounded(got, want, rmsnorm_bound(x64, s, dy64, C) + 2 * U * want.abs(), "dx")


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_qknorm_rope_vjp

def qk_rope64(q, k, S, pos, freqs, R, eps):
    """the oracle's cosine_sim_scale with a scale per (row, head) S [rows, nh] and apply_rope on the first R columns of each head, column
    j < R/2 turning with j + R/2 by (j < R/4 ? pos_y : pos_x) freqs[h, j]"""
    rows, nh, e = q.shape
    T = pos.shape[0]
    p = pos[torch.arange(rows, device=q.device) % T]
    j = torch.arange(R // 2, device=q.device)
    theta = torch.where(j < R // 4, p[:, None, 0:1], p[:, None, 1:2]) * freqs[None]      # [rows, nh, R/2]
    sq = S.sqrt()[..., None]
    q = q * (sq * torch.rsqrt((q ** 2).sum(-1, keepdim=True) + eps))
    k = k * (sq * torch.rsqrt((k ** 2).sum(-1, keepdim=True) + eps))
    return O.apply_rope(q, theta), O.apply_rope(k, theta)


def rope_abs(v, R):
    """|v_j| + |v_pair(j)| on the rotated columns, |v_j| on the rest: the magnitude a rotation's roundings scale with"""
    a = v.abs()
    out = a.clone()
    out[..., :R // 2] += a[..., R // 2:R]
    out[..., R // 2:R] += a[..., :R // 2]
    return out


# (B, T, nh, e, R, eps, dscale): d_head 16, 32, 64 and 128 with image_transformer_v2's R = e / 2 and eps 1e-6, and image_transformer_v1's R = e
# and eps e 1e-6; config_cifar10's level 0 at B = 64 (16384 rows, 4 heads of 64)
QK = [(3, 16, 2, 16, 8, 1e-6, True), (2, 12, 3, 32, 16, 1e-6, False), (3, 16, 2, 64, 32, 1e-6, True), (1, 9, 1, 128, 64, 1e-6, True),
      (2, 16, 4, 64, 64, 64e-6, True), (3, 7, 2, 32, 32, 32e-6, False), (1, 5, 2, 128, 128, 128e-6, True), (64, 256, 4, 64, 32, 1e-6, True)]


@pytest.mark.parametrize("B,T,nh,e,R,eps,with_dscale", QK)
def test_qknorm_rope_vjp(B, T, nh, e, R, eps, with_dscale):
    g = _gen("qk", B, T, nh, e, R)
    rows = B * T
    qkv = torch.randn(rows, 3, nh, e, device=DEV, generator=g) * 1.5
    dq = torch.randn(rows, 3, nh, e, device=DEV, generator=g)
    side = math.isqrt(T) + 1
    pos = (torch.rand(T, 2, device=DEV, generator=g) * 2 - 1) * (side / (side + 1))
    freqs = torch.rand(nh, R // 2, device=DEV, generator=g) * 9 * math.pi + math.pi
    scale = torch.rand(nh, device=DEV, generator=g) * 9 + 1

    def run():
        n = dq.numel()
        buf, d = _tail(n)
        d.copy_(dq.flatten())
        dsbuf, ds = _guarded(rows * nh) if with_dscale else (None, None)
        got, dsg = _native.qknorm_rope_vjp(qkv, d.view(dq.shape), pos, freqs, scale, eps, R, None if ds is None else ds.view(rows, nh))
        assert (buf[n:] == SENTINEL).all(), "a write past the end of dqkv"
        if with_dscale:
            _assert_written(dsbuf, rows * nh)
        assert torch.equal(got[:, 2], dq[:, 2]), "the v third was changed"
        return got, dsg

    got, ds = run()
    again, ds2 = run()
    assert torch.equal(got, again) and (ds is None or torch.equal(ds, ds2)), "two calls differ"
    q64, k64, dq64, dk64 = qkv[:, 0].double(), qkv[:, 1].double(), dq[:, 0].double(), dq[:, 1].double()
    S = scale.double()[None].expand(rows, nh).contiguous()
    _, pull = torch.func.vjp(lambda a, b, s: qk_rope64(a, b, s, pos.double(), freqs.double(), R, eps), q64, k64, S)
    wq, wk, wS = pull((dq64, dk64))
    sqs = scale.double().sqrt()[None, :, None]
    terms = []
    for v, d in ((q64, dq64), (k64, dk64)):
        rho = torch.rsqrt((v * v).sum(-1, keepdim=True) + eps)
        G = rope_abs(d, R)
        terms.append((v, rho, G))
    for t, want in ((0, wq), (1, wk)):
        v, rho, G = terms[t]
        bound = (e + 24) * U * sqs * (rho * G + v.abs() * rho ** 3 * (v.abs() * G).sum(-1, keepdim=True))
        _assert_bounded(got[:, t], want, bound, "dq" if t == 0 else "dk")
    if with_dscale:
        mag = sum((v.abs() * G).sum(-1) * rho[..., 0] for v, rho, G in terms) / (2 * sqs[..., 0])
        _assert_bounded(ds, wS, (e + 24) * U * mag, "dscale rows")


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_geglu_vjp

def geglu64(h):
    """the oracle's linear_geglu after its projection: value * gelu(gate)"""
    a, gate = h.chunk(2, dim=-1)
    return a * F.gelu(gate)


# (M, F): one element, ragged sizes, and config_mnist's / config_cifar10's feed-forward at B = 64, 4 to 48 passes of the grid
@pytest.mark.parametrize("M,Fd", [(1, 1), (7, 33), (9, 96), (3136, 768), (16384, 768), (4096, 1536)])
def test_geglu_vjp(M, Fd):
    g = _gen("geglu", M, Fd)
    h = torch.randn(M, 2 * Fd, device=DEV, generator=g) * 2
    dy = torch.randn(M, Fd, device=DEV, generator=g)
    buf, out = _guarded(M * 2 * Fd)
    got = _native.geglu_vjp(h, dy, out=out.view(M, 2 * Fd))
    _assert_written(buf, M * 2 * Fd)
    assert torch.equal(got, _native.geglu_vjp(h, dy)), "two calls differ"
    h64, dy64 = h.double(), dy.double()
    _, pull = torch.func.vjp(geglu64, h64)
    want = pull(dy64)[0]
    a, gate = h64.chunk(2, dim=-1)
    Phi = 0.5 * (1 + torch.erf(gate / math.sqrt(2)))
    phi = torch.exp(-0.5 * gate * gate) / math.sqrt(2 * math.pi)
    b_val = 8 * U * dy64.abs() * (gate.abs() + 1)                                            # erf's absolute error through g Phi
    b_gate = 8 * U * (dy64 * a).abs() * (1 + Phi + (gate * gate + 4) * (gate * phi).abs())   # exp's argument, then g phi
    _assert_bounded(got, want, torch.cat([b_val, b_gate], -1), "dh")
    assert M * Fd < GRID_STRIDE or M * Fd > 4 * GRID_STRIDE


# ---------------------------------------------------------------------------------------------------------------------------------------
# TokenSplit and TokenMerge's elementwise halves

# (B, H, W, C): the smallest fine grid, ragged channels, config_mnist-sized and config_cifar10's level 0 at B = 64 (8 passes of the grid)
SPLIT = [(1, 2, 2, 1), (2, 6, 10, 7), (3, 14, 14, 33), (64, 16, 16, 256)]
FACS = [0.3, 0.5, 0.7, -0.75, 1.5]


def _coarse_to_fine(y):
    B, h, w, C4 = y.shape
    return y.view(B, h, w, 2, 2, C4 // 4).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * h, 2 * w, C4 // 4)


def _fine_to_coarse(x):
    B, H, W, C = x.shape
    return x.view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4 * C)


def test_split_cases_reach_the_grid_stride_loop():
    assert max(B * H * W * C for B, H, W, C in SPLIT) > 4 * GRID_STRIDE


@pytest.mark.parametrize("fac", FACS)
@pytest.mark.parametrize("B,H,W,C", SPLIT)
def test_split_vjp_gather_bits(B, H, W, C, fac):
    """out = patch2x2(fac dup), dup *= 1 - fac in place: torch's fp32 products on the GPU, bit for bit"""
    g = _gen("split_vjp", B, H, W, C)
    dup = torch.randn(B, H, W, C, device=DEV, generator=g)
    f = torch.tensor([fac], device=DEV)
    n = dup.numel()

    def run():
        dbuf, d = _tail(n)
        d.copy_(dup.flatten())
        obuf, out = _guarded(n)
        got = _native.split_vjp_gather(d.view(dup.shape), f, out=out.view(B, H // 2, W // 2, 4 * C))
        _assert_written(obuf, n)
        assert (dbuf[n:] == SENTINEL).all(), "a write past the end of dup"
        return got, d.view(dup.shape)

    got, dnew = run()
    again, dnew2 = run()
    assert torch.equal(got, again) and torch.equal(dnew, dnew2), "two calls differ"
    assert torch.equal(got, _fine_to_coarse(f * dup))
    assert torch.equal(dnew, (1 - f) * dup)


@pytest.mark.parametrize("fac", FACS)
@pytest.mark.parametrize("B,H,W,C", SPLIT)
def test_split_unpatch_lerp_is_torch_lerp(B, H, W, C, fac):
    """up = torch.lerp(skip, unpatch2x2(y), fac) bit for bit, with fac a 0-dim tensor as TokenSplit's parameter: both of ATen's branches
    (|fac| < 0.5 and not), fac < -0.5 and fac > 1 among them"""
    g = _gen("split_lerp", B, H, W, C)
    y = torch.randn(B, H // 2, W // 2, 4 * C, device=DEV, generator=g)
    skip = torch.randn(B, H, W, C, device=DEV, generator=g)
    f = torch.tensor([fac], device=DEV)
    n = skip.numel()
    buf, out = _guarded(n)
    got = _native.split_unpatch_lerp(y, skip, f, out=out.view(skip.shape))
    _assert_written(buf, n)
    assert torch.equal(got, _native.split_unpatch_lerp(y, skip, f)), "two calls differ"
    want = torch.lerp(skip, _coarse_to_fine(y), f.view(()))
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} of {n} elements differ from torch.lerp, e.g. {got[bad][:3].tolist()} vs {want[bad][:3].tolist()}"


@pytest.mark.parametrize("B,H,W,C", SPLIT)
def test_merge_scatter_add_bits(B, H, W, C):
    g = _gen("merge_add", B, H, W, C)
    d = torch.randn(B, H // 2, W // 2, 4 * C, device=DEV, generator=g)
    start = torch.randn(B, H, W, C, device=DEV, generator=g)
    n = start.numel()
    buf, out = _tail(n)
    out.copy_(start.flatten())
    got = _native.merge_scatter_add(d, out.view(start.shape))
    assert (buf[n:] == SENTINEL).all(), "a write past the end of dfine"
    assert torch.equal(got, _native.merge_scatter_add(d, start.clone())), "two calls differ"
    assert torch.equal(got, start + _coarse_to_fine(d))


# ---------------------------------------------------------------------------------------------------------------------------------------
# patch_out and patch_in

def patch_out64(tokens, scale, w, B, H, W, ph, pw):
    """out_norm then patch_out as the oracle's model_forward ends: tokens [T, C0] -> [B, C, H, W]"""
    x = O.rms_norm(tokens.view(B, H // ph, W // pw, -1), scale)
    return O.token_split(x, w, ph, pw).movedim(-1, -3)


def _patch_rows(img, ph, pw):
    B, C, H, W = img.shape
    return img.view(B, C, H // ph, ph, W // pw, pw).permute(0, 2, 4, 3, 5, 1).reshape(B * (H // ph) * (W // pw), ph * pw * C)


# (B, C, H, W, ph, pw, C0): tiny, non-square patches with ragged widths, config_mnist at B = 64 (4 x 4 patches of 1 channel, 256 wide) and
# config_cifar10 at B = 64 (2 x 2 of 3, 256)
PATCH = [(1, 1, 4, 4, 4, 4, 4), (2, 3, 8, 12, 2, 4, 33), (3, 1, 12, 6, 4, 2, 96), (64, 1, 28, 28, 4, 4, 256), (64, 3, 32, 32, 2, 2, 256)]


@pytest.mark.parametrize("sd", [0.0, 0.5], ids=["raw", "karras"])
@pytest.mark.parametrize("B,C,H,W,ph,pw,C0", PATCH)
def test_patch_out_vjp(B, C, H, W, ph, pw, C0, sd):
    """dnorm = patch(c_out u) W bit for bit on integers (raw model); dtokens, dnorm and rstd within their fp32 bounds on normal operands"""
    g = _gen("patch_out", B, C, H, W, ph, pw, C0)
    T, N = B * (H // ph) * (W // pw), ph * pw * C
    sigma = torch.exp(torch.randn(B, device=DEV, generator=g))
    tokens = torch.randn(T, C0, device=DEV, generator=g) * 2 + 0.3
    scale = torch.randn(C0, device=DEV, generator=g) + 1

    def run(w, u):
        bufs = [_guarded(n) for n in (T * C0, T * C0, T)]
        got = _native.patch_out_vjp(tokens, scale, w, u, (ph, pw), sigma=sigma, sigma_data=sd, out=bufs[0][1].view(T, C0),
                                    dnorm=bufs[1][1].view(T, C0), rstd=bufs[2][1])
        for buf, v in bufs:
            _assert_written(buf, v.numel())
        again = _native.patch_out_vjp(tokens, scale, w, u, (ph, pw), sigma=sigma, sigma_data=sd, dnorm=torch.empty(T, C0, device=DEV),
                                      rstd=torch.empty(T, device=DEV))
        assert all(torch.equal(a, b) for a, b in zip(got, again)), "two calls differ"
        return got

    if sd == 0:
        w, u = _ints((N, C0), g), _ints((B, C, H, W), g)
        _, dnorm, _ = run(w, u)
        _assert_exact(dnorm, _patch_rows(u, ph, pw).double().cpu() @ w.double().cpu())
    w, u = torch.randn(N, C0, device=DEV, generator=g), torch.randn(B, C, H, W, device=DEV, generator=g)
    dtok, dnorm, rstd = run(w, u)
    c_out = O.karras_scalings(sigma.double(), sd)[1].view(-1, 1, 1, 1) if sd > 0 else torch.ones(B, 1, 1, 1, device=DEV, dtype=torch.float64)
    cu = c_out * u.double()
    x64, s64 = tokens.double(), scale.double()
    _, pull = torch.func.vjp(lambda t: patch_out64(t, s64, w.double(), B, H, W, ph, pw), x64)
    want = pull(cu)[0]
    dn_mag = _patch_rows(cu.abs(), ph, pw) @ w.double().abs()
    _assert_bounded(dnorm, _patch_rows(cu, ph, pw) @ w.double(), (N + 8) * U * dn_mag, "dnorm")
    r = torch.rsqrt((x64 * x64).mean(-1) + 1e-6)
    _assert_bounded(rstd, r, (C0 / 2 + 4) * U * r, "rstd")
    bound = rmsnorm_bound(x64, s64, dn_mag, C0 + N + 8)
    _assert_bounded(dtok, want, bound, "dtokens")


@pytest.mark.parametrize("Cout,ph,pw", [(3, 4, 4), (1, 4, 4), (3, 2, 2)])
def test_patch_out_vjp_shared_memory_edge(Cout, ph, pw):
    """4 (C0 + ph pw Cout) floats of shared memory, at most 48 KiB: the widest C0 runs and matches, the next one returns
    KDB_ERR_UNSUPPORTED and launches nothing"""
    N = ph * pw * Cout
    widest = 12288 // 4 - N
    assert 4 * (widest + N) <= 12288 < 4 * (widest + 1 + N)
    g = _gen("patch_out_edge", Cout, ph, pw)
    B, H, W = 1, 2 * ph, ph * pw
    T = B * (H // ph) * (W // pw)
    for C0 in (widest, widest + 1):
        tokens, scale = torch.randn(T, C0, device=DEV, generator=g), torch.randn(C0, device=DEV, generator=g) + 1
        w, u = _ints((N, C0), g), _ints((B, Cout, H, W), g)
        buf, out = _guarded(T * C0)
        dn = torch.full((T, C0), float("nan"), device=DEV)
        torch.cuda.synchronize()
        n0 = _native.launch_count()
        if C0 == widest:
            dtok, dnorm, _ = _native.patch_out_vjp(tokens, scale, w, u, (ph, pw), out=out.view(T, C0), dnorm=dn)
            _assert_written(buf, T * C0)
            _assert_exact(dnorm, _patch_rows(u, ph, pw).double().cpu() @ w.double().cpu())
        else:
            with pytest.raises(RuntimeError, match="-2"):
                _native.patch_out_vjp(tokens, scale, w, u, (ph, pw), out=out.view(T, C0), dnorm=dn)
            torch.cuda.synchronize()
            assert _native.launch_count() == n0 and out.isnan().all() and dn.isnan().all()


# (B, C, H, W, ph, pw, N): non-square patches, config_mnist and config_cifar10 at B = 64, and 786,432 pixels (past one pass of the grid)
PATCH_IN = [(1, 1, 4, 4, 4, 4, 4), (2, 3, 8, 12, 2, 4, 33), (3, 1, 12, 6, 4, 2, 96), (64, 1, 28, 28, 4, 4, 256), (64, 3, 32, 32, 2, 2, 256),
            (64, 3, 64, 64, 4, 2, 64)]


def test_patch_in_cases_reach_the_grid_stride_loop():
    assert max(B * C * H * W for B, C, H, W, *_ in PATCH_IN) > GRID_STRIDE


@pytest.mark.parametrize("sd", [0.0, 0.5], ids=["raw", "karras"])
@pytest.mark.parametrize("B,C,H,W,ph,pw,N", PATCH_IN)
def test_patch_in_vjp(B, C, H, W, ph, pw, N, sd):
    """unpatch(dtokens W) bit for bit on integers (raw model); with the Karras scalings c_skip u + c_in unpatch(dtokens W) within its bound"""
    g = _gen("patch_in", B, C, H, W, ph, pw, N)
    T, K = B * (H // ph) * (W // pw), ph * pw * C
    sigma = torch.exp(torch.randn(B, device=DEV, generator=g))
    size = (B, C, H, W)

    def run(dt, w, u):
        buf, out = _guarded(B * C * H * W)
        got = _native.patch_in_vjp(dt, w, size, (ph, pw), u=u, sigma=sigma, sigma_data=sd, out=out.view(size))
        _assert_written(buf, out.numel())
        assert torch.equal(got, _native.patch_in_vjp(dt, w, size, (ph, pw), u=u, sigma=sigma, sigma_data=sd)), "two calls differ"
        return got

    def merge64(dt, w, u):
        """the input gradient of c_skip x + F(c_in x) with F's first op the oracle's token_merge of x [B, C, H, W]"""
        c_skip, _, c_in = (c.view(-1, 1, 1, 1) for c in O.karras_scalings(sigma.double(), sd)) if sd > 0 else (0, 1, 1)
        x0 = torch.zeros(size, device=DEV, dtype=torch.float64)
        _, pull = torch.func.vjp(lambda x: O.token_merge((x * c_in).movedim(-3, -1), w, ph, pw), x0)
        return pull(dt.view(B, H // ph, W // pw, N))[0] + (c_skip * u if sd > 0 else 0)

    if sd == 0:
        dt, w = _ints((T, N), g), _ints((N, K), g)
        _assert_exact(run(dt, w, None), merge64(dt.double(), w.double(), None).cpu())
    dt, w, u = torch.randn(T, N, device=DEV, generator=g), torch.randn(N, K, device=DEV, generator=g), torch.randn(size, device=DEV, generator=g)
    got = run(dt, w, u)
    want = merge64(dt.double(), w.double(), u.double())
    mag = merge64(dt.double().abs(), w.double().abs(), u.double().abs())
    _assert_bounded(got, want, (N + 6) * U * mag, "grad_x")


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_model_mapping_vjp

def mapping_model(mw, depth, dff, classes, mcond):
    spec = {"model": {"type": "image_transformer_v2", "input_channels": 1, "input_size": [8, 8], "patch_size": [2, 2], "depths": [1],
                      "widths": [32], "d_ffs": [64], "mapping_width": mw, "mapping_depth": depth, "mapping_d_ff": dff,
                      "mapping_cond_dim": mcond, "self_attns": [{"type": "global", "d_head": 16}]},
            "dataset": {"num_classes": 10 if classes else 0}}
    _, inner, sd, _ = build(spec)
    return inner.engine(), {k: v.double().to(DEV) for k, v in sd.items()}


def check_mapping_vjp(eng, sd, sigma, aug, cls, mc, dcond, mw, depth, dff):
    """kdb_model_mapping_vjp stage by stage against float64: each activation and gradient against the oracle's op (or torch.func.vjp of it)
    at the kernel's own previous values, within the fp32 roundings of that stage; then demb against the vjp of the whole network"""
    rows = sigma.numel()
    L = _native.mapping_layout(mw, dff, depth)
    kbuf, keep = _guarded(rows * L["keep"])
    gbuf, grad = _guarded(rows * L["grad"])
    keep, grad = eng.mapping_vjp(sigma, dcond, aug, cls, mc, out=(keep.view(rows, -1), grad.view(rows, -1)))
    assert (kbuf[keep.numel():] == SENTINEL).all() and (gbuf[grad.numel():] == SENTINEL).all(), "a write past the end of keep or grad"
    k2, g2 = eng.mapping_vjp(sigma, dcond, aug, cls, mc)
    written = torch.ones(L["keep"], dtype=torch.bool, device=DEV)
    for l in range(depth):   # the GEGLU output's padding to a multiple of 4 floats is not written
        written[L["g"](l) + dff:L["xn"](l + 1) if l + 1 < depth else L["keep"]] = False
    assert not keep[:, written].isnan().any() and not grad.isnan().any(), "an activation or gradient was left unwritten"
    assert torch.equal(keep[:, written], k2[:, written]) and torch.equal(grad, g2), "two calls differ"
    K, G = keep.double(), grad.double()
    kv = lambda off, n: K[:, off:off + n]
    gv = lambda off, n: G[:, off:off + n]
    W = lambda k: sd[k]
    half = mw // 2
    two_pi = 2 * math.pi
    checks = []
    # Fourier features of log(sigma) / 4 and of aug_cond (zeros without it)
    arg_t = two_pi * (sigma.double().log() / 4)[:, None] * W("time_emb.weight")[:, 0][None]
    checks.append(("ff_t", kv(L["ff_t"], mw), torch.cat([arg_t.cos(), arg_t.sin()], 1), (6 * arg_t.abs() + 4).repeat(1, 2) * U))
    a64 = aug.double() if aug is not None else torch.zeros(rows, 9, device=DEV, dtype=torch.float64)
    arg_a = two_pi * a64 @ W("aug_emb.weight").T
    mag_a = two_pi * a64.abs() @ W("aug_emb.weight").abs().T
    checks.append(("ff_a", kv(L["ff_a"], mw), torch.cat([arg_a.cos(), arg_a.sin()], 1), (14 * mag_a + 4).repeat(1, 2) * U))
    # the summed embedding from the kernel's features
    ff_t, ff_a = kv(L["ff_t"], mw), kv(L["ff_a"], mw)
    emb = ff_t @ W("time_in_proj.weight").T + ff_a @ W("aug_in_proj.weight").T
    mag = ff_t.abs() @ W("time_in_proj.weight").abs().T + ff_a.abs() @ W("aug_in_proj.weight").abs().T
    if cls is not None:
        emb, mag = emb + W("class_emb.weight")[cls], mag + W("class_emb.weight")[cls].abs()
    if mc is not None:
        emb = emb + mc.double() @ W("mapping_cond_in_proj.weight").T
        mag = mag + mc.double().abs() @ W("mapping_cond_in_proj.weight").abs().T
    checks.append(("emb", kv(L["emb"], mw), emb, (mw + (mc.shape[1] if mc is not None else 0) + 8) * U * mag))
    # the forward of in_norm and each block from the kernel's previous activations
    norm = lambda x, s: O.rms_norm(x, s)
    checks.append(("r0", kv(L["r"](0), mw), norm(kv(L["emb"], mw), W("mapping.in_norm.scale")), (mw + 8) * U * kv(L["r"](0), mw).abs()))
    for l in range(depth):
        p = f"mapping.blocks.{l}."
        r, xn, up, gg = kv(L["r"](l), mw), kv(L["xn"](l), mw), kv(L["up"](l), 2 * dff), kv(L["g"](l), dff)
        checks.append((f"xn{l}", xn, norm(r, W(p + "norm.scale")), (mw + 8) * U * xn.abs()))
        checks.append((f"up{l}", up, xn @ W(p + "up_proj.weight").T, (mw + 2) * U * (xn.abs() @ W(p + "up_proj.weight").abs().T)))
        a, gate = up.chunk(2, -1)
        checks.append((f"g{l}", gg, a * F.gelu(gate), 8 * U * a.abs() * (gate.abs() + 1)))
        checks.append((f"r{l + 1}", kv(L["r"](l + 1), mw), r + gg @ W(p + "down_proj.weight").T,
                       (dff + 2) * U * (r.abs() + gg.abs() @ W(p + "down_proj.weight").abs().T)))
    # the reverse walk from the kernel's gradients
    dc = dcond.double()
    rD = kv(L["r"](depth), mw)
    s = W("mapping.out_norm.scale")
    checks.append(("dr_out", gv(L["dr"](depth), mw), torch.func.vjp(lambda x: norm(x, s), rD)[1](dc)[0], rmsnorm_bound(rD, s, dc, mw)))
    for l in reversed(range(depth)):
        p = f"mapping.blocks.{l}."
        dr1, up, r = gv(L["dr"](l + 1), mw), kv(L["up"](l), 2 * dff), kv(L["r"](l), mw)
        Wd, Wu, s = W(p + "down_proj.weight"), W(p + "up_proj.weight"), W(p + "norm.scale")
        dg, dg_mag = dr1 @ Wd, dr1.abs() @ Wd.abs()
        a, gate = up.chunk(2, -1)
        slope = 0.5 * (1 + torch.erf(gate / math.sqrt(2))) + gate * torch.exp(-0.5 * gate * gate) / math.sqrt(2 * math.pi)
        want_dh = torch.func.vjp(geglu64, up)[1](dg)[0]
        b_dh = torch.cat([(mw + 2) * U * dg_mag * (F.gelu(gate).abs() + gate.abs() * 8 * U) + 8 * U * dg.abs() * (gate.abs() + 1),
                          (mw + 2) * U * dg_mag * (a * slope).abs() + 8 * U * (dg * a).abs() * (2 + (gate * gate + 4))], -1)
        checks.append((f"dh{l}", gv(L["dh"](l), 2 * dff), want_dh, b_dh))
        dh = gv(L["dh"](l), 2 * dff)
        checks.append((f"dxn{l}", gv(L["dxn"](l), mw), dh @ Wu, (2 * dff + 2) * U * (dh.abs() @ Wu.abs())))
        dxn = gv(L["dxn"](l), mw)
        want = dr1 + torch.func.vjp(lambda x: norm(x, s), r)[1](dxn)[0]
        checks.append((f"dr{l}", gv(L["dr"](l), mw), want, rmsnorm_bound(r, s, dxn, mw) + 2 * U * (dr1.abs() + want.abs())))
    e0, s = kv(L["emb"], mw), W("mapping.in_norm.scale")
    dr0 = gv(L["dr"](0), mw)
    checks.append(("demb", gv(L["demb"], mw), torch.func.vjp(lambda x: norm(x, s), e0)[1](dr0)[0], rmsnorm_bound(e0, s, dr0, mw)))
    for name, got, want, bound in checks:
        _assert_bounded(got, want, bound, name)
    # and the whole backward at once: demb against torch.func.vjp of the oracle's mapping network from the float64 embedding
    net = lambda x: O.mapping_network(sd, x)
    want = torch.func.vjp(net, emb)[1](dc)[0]
    err = (gv(L["demb"], mw) - want).norm() / want.norm()
    assert err <= 2e-5 * (depth + 1), f"demb: relative error {err:.3e} against the whole network's vjp"


# (mw, depth, d_ff): mw 64 (block_matvec's scalar loads) and 256 (float4 loads), d_ff 98 (GEGLU outputs padded to 100 floats) and 768
@pytest.mark.parametrize("rows", [1, 64])
@pytest.mark.parametrize("conds", ["none", "class+mapping_cond+aug"])
@pytest.mark.parametrize("depth", [1, 2, 8])
@pytest.mark.parametrize("mw,dff", [(64, 98), (256, 768)])
def test_mapping_vjp_against_float64(mw, dff, depth, conds, rows):
    full = conds != "none"
    mcond = 12 if full else 0
    eng, sd = mapping_model(mw, depth, dff, full, mcond)
    g = _gen("mapping", mw, depth, conds, rows)
    sigma = torch.exp(torch.randn(rows, device=DEV, generator=g) * 1.5)
    aug = torch.randn(rows, 9, device=DEV, generator=g) * 0.3 if full else None
    cls = torch.randint(0, 11, (rows,), device=DEV, generator=g) if full else None
    mc = torch.randn(rows, mcond, device=DEV, generator=g) if full else None
    dcond = torch.randn(rows, mw, device=DEV, generator=g)
    check_mapping_vjp(eng, sd, sigma, aug, cls, mc, dcond, mw, depth, dff)
