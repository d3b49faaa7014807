"""The U-Net's backward kernels one by one against float64 torch.func, at the edges a whole-model tolerance cannot see: the convolution's
weight gradient and (the forward convolution on the flipped weight) input gradient at the zero-padded borders, with one and two sources, ks 1
and 3, on 7x7, 8x8 and odd non-square grids with N not a multiple of 64, and at training shapes whose weight-gradient row chunks end inside an
image and a pixel row, with a short last chunk; the AdaGN (+ GELU) backward with groups that straddle the two sources, group widths past the
CTA's 8 warps and its mapper-output rows; the resampling adjoints at the reflect borders, their adjointness and `add` aliased to the output;
pixel_unshuffle, proj_out's input gradient and the mapping network's backward, with its shared-memory edge.

Integer-valued operands, where the arithmetic is exact, must match bit for bit; random normal ones stay within an element-wise fp32 bound
computed from float64 sums of |terms|.  Outputs start as NaN with a sentinel tail (unwritten elements and writes past the end both show), and
two calls give the same bits."""
import math

import pytest
import torch
from torch.nn import functional as F

from oracle import unet_oracle as U
from test_gpu_train_kernels import U as EPS, _assert_written, _chunks, _guarded

from k_diffusion import _native

pytestmark = pytest.mark.gpu
DEV = "cuda"

GRIDS = [(7, 7), (8, 8), (5, 9)]


def ints(g, *shape, lo=-3, hi=4):
    return torch.randint(lo, hi, shape, generator=g).double()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def conv64(x1, x2, w, ks):
    """torch's conv2d (zero padding ks // 2) on token-major [B, h, w, c] inputs, float64, -> token-major"""
    x = torch.cat([x1, x2], -1) if x2 is not None else x1
    return F.conv2d(nchw(x), w, padding=ks // 2).permute(0, 2, 3, 1)


def tap_major(w):
    n, c, k, _ = w.shape
    return w.permute(0, 2, 3, 1).reshape(n, k * k, c).contiguous()


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("ks", [1, 3])
@pytest.mark.parametrize("c2", [0, 8])
def test_conv_wgrad_and_dgrad_exact_on_integers(grid, ks, c2):
    g = torch.Generator().manual_seed(ks * 10 + c2)
    B, (h, w), c1, N = 2, grid, 12, 20
    x1, x2 = ints(g, B, h, w, c1), (ints(g, B, h, w, c2) if c2 else None)
    dy = ints(g, B, h, w, N)
    wt = ints(g, N, c1 + c2, ks, ks)
    xs = (x1,) if x2 is None else (x1, x2)
    _, pull = torch.func.vjp(lambda wt_, *xx: conv64(xx[0], xx[1] if len(xx) > 1 else None, wt_, ks), wt, *xs)
    dw_want, *dx_want = pull(dy)
    dw = _native.unet_conv_wgrad(dy.float().to(DEV), x1.float().to(DEV), ks, None if x2 is None else x2.float().to(DEV))
    assert torch.equal(dw.cpu().double(), dw_want)
    # the input gradient: the forward convolution of dy with w'[c, tap, n] = w[n, c, flipped tap]
    wflip = _native.unet_flip_conv_weight(tap_major(wt).float().to(DEV))
    assert torch.equal(wflip.cpu().double(), tap_major(wt.flip(2, 3).transpose(0, 1)))
    dx = _native.unet_conv(dy.float().to(DEV).contiguous(), wflip, ks).cpu().double()
    assert torch.equal(dx, torch.cat(dx_want, -1))


@pytest.mark.parametrize("grid", GRIDS)
def test_conv_wgrad_random_within_the_fp32_bound(grid):
    g = torch.Generator().manual_seed(1)
    B, (h, w), N = 3, grid, 36
    x1, x2, dy = (torch.randn(B, h, w, c, generator=g).double() for c in (16, 20, N))
    wt = torch.zeros(N, 36, 3, 3, dtype=torch.float64)
    _, pull = torch.func.vjp(lambda wt_: conv64(x1, x2, wt_, 3), wt)
    (want,) = pull(dy)
    got = _native.unet_conv_wgrad(dy.float().to(DEV), x1.float().to(DEV), 3, x2.float().to(DEV)).cpu().double()
    bound = 2 * B * h * w * 2 ** -24 * torch.einsum("bhwn,bhwc->nc", dy.abs(), torch.cat([x1, x2], -1).abs()).max()
    assert (got - want).abs().max() <= bound
    assert torch.equal(got, _native.unet_conv_wgrad(dy.float().to(DEV), x1.float().to(DEV), 3, x2.float().to(DEV)).cpu().double())


# (B, h, w, c1, c2, N, ks) whose weight gradient takes several wgrad_chunk row chunks: B = 3 on 9x13 splits 351 rows as 176 + 175, the
# boundary at image 1, pixel row 4, column 7; the others run 3, 4 and 13 chunks with a short last one, and config_cifar10's level-0 conv at B = 8
TRAIN_CONVS = [(3, 9, 13, 12, 8, 20, 3), (3, 9, 13, 20, 0, 20, 1), (5, 10, 11, 8, 8, 36, 3), (7, 12, 12, 16, 0, 64, 1), (8, 20, 20, 8, 4, 8, 1),
               (8, 32, 32, 128, 0, 128, 3)]


def _conv_chunks(B, h, w, c, N, ks):
    return _chunks(B * h * w, N, c * ks * ks)


def test_train_conv_cases_reach_several_chunks_and_a_short_last_one():
    """wgrad_chunk's arithmetic on TRAIN_CONVS: every case runs several chunks; the first ends inside an image and inside a pixel row with a
    short last chunk; a short last chunk and a boundary inside a pixel row occur with one and with two sources, and with ks 1 and 3"""
    short, mid_row = set(), set()
    for B, h, w, c1, c2, N, ks in TRAIN_CONVS:
        chunk, count, last = _conv_chunks(B, h, w, c1 + c2, N, ks)
        assert count > 1, (B, h, w, c1, c2, N, ks)
        if last < chunk:
            short |= {("two" if c2 else "one", ks)}
        if chunk % (h * w) and chunk % w:
            mid_row |= {("two" if c2 else "one", ks)}
    assert _conv_chunks(3, 9, 13, 20, 20, 3) == (176, 2, 175)
    assert short >= {("one", 1), ("two", 3)} and mid_row >= {("one", 1), ("two", 3)}, (short, mid_row)


@pytest.mark.parametrize("B,h,w,c1,c2,N,ks", TRAIN_CONVS)
def test_conv_wgrad_and_dgrad_at_training_shapes(B, h, w, c1, c2, N, ks):
    """The weight gradient over several row chunks: bit for bit on integers (every partial sum stays below 2^24), within the fp32 bound on
    normal operands; the input gradient (unet_conv on the flipped weight) within its bound"""
    g = torch.Generator().manual_seed(B * 1000 + h * w + c1 + c2 + N + ks)
    C = c1 + c2
    wt = torch.zeros(N, C, ks, ks, dtype=torch.float64)

    def run_wgrad(dy, x1, x2):
        f = lambda t: t.float().to(DEV).contiguous()
        buf, out = _guarded(N * C * ks * ks)
        got = _native.unet_conv_wgrad(f(dy), f(x1), ks, None if x2 is None else f(x2), out=out.view(N, C, ks, ks))
        _assert_written(buf, out.numel())
        assert torch.equal(got, _native.unet_conv_wgrad(f(dy), f(x1), ks, None if x2 is None else f(x2))), "two calls differ"
        return got.cpu().double()

    def split(x):
        return (x[..., :c1], x[..., c1:]) if c2 else (x, None)

    x, dy = ints(g, B, h, w, C), ints(g, B, h, w, N)
    _, pull = torch.func.vjp(lambda wt_: conv64(x, None, wt_, ks), wt)
    assert torch.equal(run_wgrad(dy, *split(x)), pull(dy)[0])
    x, dy = torch.randn(B, h, w, C, generator=g).double(), torch.randn(B, h, w, N, generator=g).double()
    x, dy = x.float().double(), dy.float().double()
    _, pull = torch.func.vjp(lambda wt_: conv64(x, None, wt_, ks), wt)
    _, pull_abs = torch.func.vjp(lambda wt_: conv64(x.abs(), None, wt_, ks), wt)
    M = B * h * w
    got = run_wgrad(dy, *split(x))
    bound = 1.01 * (M + _conv_chunks(B, h, w, C, N, ks)[1]) * EPS * pull_abs(dy.abs())[0]
    err = (got - pull(dy)[0]).abs()
    assert (err <= bound).all(), f"weight gradient: max error {err.max():.3e}, worst excess {(err - bound).max():.3e}"
    # the input gradient: the forward convolution of dy with the flipped weight, every output element within N k k terms' bound
    wt = torch.randn(N, C, ks, ks, generator=g).float().double()
    _, pull = torch.func.vjp(lambda xx: conv64(xx, None, wt, ks), x)
    _, pull_abs = torch.func.vjp(lambda xx: conv64(xx, None, wt.abs(), ks), x)
    wflip = _native.unet_flip_conv_weight(tap_major(wt).float().to(DEV))
    buf, out = _guarded(M * C)
    dx = _native.unet_conv(dy.float().to(DEV).contiguous(), wflip, ks, out=out.view(B, h, w, C))
    _assert_written(buf, M * C)
    assert torch.equal(dx, _native.unet_conv(dy.float().to(DEV).contiguous(), wflip, ks)), "two calls differ"
    bound = 1.01 * (N * ks * ks + 2) * EPS * pull_abs(dy.abs())[0]
    err = (dx.cpu().double() - pull(dy)[0]).abs()
    assert (err <= bound).all(), f"input gradient: max error {err.max():.3e}, worst excess {(err - bound).max():.3e}"


def adagn64(x, cond, off, groups, gelu):
    C = x.shape[-1]
    wgt, bias = cond[:, off:off + C], cond[:, off + C:off + 2 * C]
    y = F.group_norm(nchw(x), groups, eps=U.GN_EPS) * (wgt + 1)[:, :, None, None] + bias[:, :, None, None]
    return (F.gelu(y) if gelu else y).permute(0, 2, 3, 1)


# (groups, c1, c2, B, h, w): one and several groups; groups straddling the in1 | in2 boundary (c1 % (C / groups) != 0: a UBlock's first
# ResConvBlock), among them 34-channel ones; group widths past the CTA's 8 warps and not multiples of 8, and of one channel; HW from 4 to 1024
ADAGN = [(1, 24, 0, 2, 5, 6), (3, 48, 0, 2, 5, 6), (2, 32, 32, 2, 5, 6), (4, 64, 64, 2, 5, 6), (2, 48, 16, 4, 3, 15), (4, 100, 36, 16, 2, 2),
         (3, 30, 30, 5, 9, 5), (1, 12, 0, 3, 32, 32), (2, 128, 128, 16, 32, 32), (8, 4, 4, 2, 1, 4)]


def test_adagn_cases_reach_the_edges():
    cg = {(c1 + c2) // groups for groups, c1, c2, *_ in ADAGN}
    straddle = [(groups, c1, c2) for groups, c1, c2, *_ in ADAGN if c2 and c1 % ((c1 + c2) // groups)]
    assert {(2, 48, 16), (4, 100, 36)} <= set(straddle) and 34 in cg
    assert any(c > 8 and c % 8 for c in cg) and 1 in cg and max(cg) > 8
    assert {h * w for *_, h, w in ADAGN} >= {4, 45, 1024} and max(B for *_, B, h, w in ADAGN) == 16


def adagn_bound(x, cond, dy, add, off, groups, gelu):
    """Element-wise bounds on the fp32 AdaGN backward's dx and its d scale, d shift rows: c u times the float64 magnitudes of the terms each
    sums, with the rounding of the group mean and rstd carried through x^ (and the GELU's slope) to every sum that reads them.  c covers the
    longest chain of roundings: a group's n = HW cg elements summed over the CTA, a channel's HW pixels, the cg channels of sa and sb."""
    B, h, w, C = x.shape
    HW, cg = h * w, C // groups
    n = HW * cg
    c = HW + cg + n / 256 + 64
    xg = x.reshape(B, HW, groups, cg)
    gmean = lambda t: t.mean(dim=(1, 3), keepdim=True)
    mu = gmean(xg)
    r = 1 / (gmean((xg - mu) ** 2) + U.GN_EPS).sqrt()
    xh = (xg - mu) * r
    wgt, bias = (t.reshape(B, 1, groups, cg) for t in (cond[:, off:off + C], cond[:, off + C:off + 2 * C]))
    s1 = (wgt + 1).abs()
    y = xh * (wgt + 1) + bias
    dyg = dy.reshape(B, HW, groups, cg)
    Sx = xh.abs() + r * gmean(xg.abs())                       # |x^| + r mean|x|: the scale of x^'s rounding
    if gelu:
        slope = 0.5 * (1 + torch.erf(y / math.sqrt(2))) + y * torch.exp(-0.5 * y * y) / math.sqrt(2 * math.pi)
        D = (dyg * slope).abs() + 0.8 * dyg.abs() * s1 * Sx + dyg.abs() * (1 + y.abs()) / 8   # |gelu''| <= 0.8; gelu_slope's own error
    else:
        D = dyg.abs()
    ds = c * EPS * (D * (xh.abs() + Sx)).sum(1)
    dt = c * EPS * D.sum(1)
    A = D * s1
    S = r * (A + gmean(A) + (xh.abs() + Sx) * gmean(A * (xh.abs() + Sx)))
    dx = c * EPS * S.reshape(B, h, w, C) + (0 if add is None else EPS * add.abs())
    return dx, torch.cat([ds.reshape(B, C), dt.reshape(B, C)], 1)


@pytest.mark.parametrize("groups,c1,c2,B,h,w", ADAGN)
@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("with_add", [False, True])
def test_adagn_vjp_against_float64(groups, c1, c2, B, h, w, gelu, with_add):
    g = torch.Generator().manual_seed(groups * 100 + c1 + c2 + B * h * w + gelu)
    C = c1 + c2
    f32 = lambda t: t.float().double()
    x = f32(torch.randn(B, h, w, C, generator=g).double() * 2 + 0.5)
    stride, off = 2 * C + 12, 8
    cond = f32(torch.randn(B, stride, generator=g).double() * 0.5)
    dy = f32(torch.randn(B, h, w, C, generator=g).double())
    add = f32(torch.randn(B, h, w, C, generator=g).double()) if with_add else None
    _, pull = torch.func.vjp(lambda xx, cc: adagn64(xx, cc, off, groups, gelu), x, cond)
    dx_want, dc_want = pull(dy)
    if add is not None:
        dx_want = dx_want + add
    dx_bound, dc_bound = adagn_bound(x, cond, dy, add, off, groups, gelu)
    f = lambda t: None if t is None else t.float().to(DEV).contiguous()
    x1, x2 = f(x[..., :c1]), (f(x[..., c1:]) if c2 else None)

    def run():
        b1, o1 = _guarded(B * h * w * c1)
        b2, o2 = _guarded(B * h * w * c2) if c2 else (None, None)
        dx1, dx2, dss = _native.unet_adagn_vjp(x1, f(dy), f(cond), off, groups, gelu, x2=x2, add=f(add),
                                               out=(o1.view(B, h, w, c1), None if o2 is None else o2.view(B, h, w, c2)))
        _assert_written(b1, o1.numel())
        if c2:
            _assert_written(b2, o2.numel())
        assert not dss[:, off:off + 2 * C].isnan().any(), "a d scale / d shift element was left unwritten"
        assert torch.isnan(dss[:, :off]).all() and torch.isnan(dss[:, off + 2 * C:]).all()   # nothing outside its rows is written
        return torch.cat([dx1, dx2], -1) if c2 else dx1, dss

    dx, dss = run()
    err = (dx.cpu().double() - dx_want).abs()
    assert (err <= dx_bound).all(), f"dx: max error {err.max():.3e}, worst excess {(err - dx_bound).max():.3e}"
    err = (dss.cpu().double()[:, off:off + 2 * C] - dc_want[:, off:off + 2 * C]).abs()
    assert (err <= dc_bound).all(), f"d scale / d shift: max error {err.max():.3e}, worst excess {(err - dc_bound).max():.3e}"
    again = run()
    assert torch.equal(again[0], dx) and torch.equal(again[1][:, off:off + 2 * C], dss[:, off:off + 2 * C]), "two calls differ"


def resample64(x, up):
    return (U.upsample if up else U.downsample)(nchw(x)).permute(0, 2, 3, 1)


# (h, w) with B = 2 and C = 6, or (h, w, B, C): the training shapes, config_cifar10's 32x32 -> 16x16 and config_mnist's 28x28 -> 14x14 -> 7x7
RESAMPLE_GRIDS = [(2, 2), (7, 7), (8, 8), (5, 9), (6, 10), (32, 32, 16, 128), (28, 28, 16, 128), (14, 14, 16, 128), (7, 7, 16, 128)]


@pytest.mark.parametrize("grid", RESAMPLE_GRIDS)
@pytest.mark.parametrize("up", [False, True])
def test_resample_vjp_exact_and_adjoint(grid, up):
    h, w, *bc = grid
    B, C = bc or (2, 6)
    g = torch.Generator().manual_seed(h * 31 + w + up + B * C)
    x = ints(g, B, h, w, C)
    y0 = resample64(x, up)
    dy = ints(g, *y0.shape)
    _, pull = torch.func.vjp(lambda xx: resample64(xx, up), x)
    (want,) = pull(dy)
    n = B * h * w * C
    buf, out = _guarded(n)
    got = _native.unet_resample_vjp(dy.float().to(DEV).contiguous(), h, w, up, out=out.view(B, h, w, C))
    _assert_written(buf, n)
    assert torch.equal(got.cpu().double(), want)
    assert torch.equal(got, _native.unet_resample_vjp(dy.float().to(DEV).contiguous(), h, w, up)), "two calls differ"
    # <resample x, y> = <x, resample^T y>
    assert torch.isclose((y0 * dy).sum(), (x * got.cpu().double()).sum(), rtol=0, atol=0)
    add = ints(g, B, h, w, C)
    got_add = _native.unet_resample_vjp(dy.float().to(DEV).contiguous(), h, w, up, add=add.float().to(DEV)).cpu().double()
    assert torch.equal(got_add, want + add)
    # add aliased to the output, as the engine's downsample adjoint adds the skip gradient in place
    out.copy_(add.float().flatten())
    _native.unet_resample_vjp(dy.float().to(DEV).contiguous(), h, w, up, add=out.view(B, h, w, C), out=out.view(B, h, w, C))
    _assert_written(buf, n)
    assert torch.equal(out.view(B, h, w, C).cpu().double(), want + add)


# pixel_unshuffle at the mnist / cifar10 shapes (B = 64, 32x32 and 28x28) and at a size past launch_unet_unshuffle's grid (grid_for: at most
# 132 * 32 CTAs of 256 threads), so that the grid-stride loop runs
UNSHUFFLE = [(64, 3, 32, 32, 1), (64, 3, 32, 32, 2), (64, 3, 32, 32, 4), (64, 1, 28, 28, 4), (64, 3, 128, 128, 1), (64, 3, 128, 128, 2),
             (16, 3, 256, 256, 4)]
GRID_THREADS = 132 * 32 * 256


def test_unshuffle_cases_reach_the_grid_stride_loop():
    for p in (1, 2, 4):
        assert any(B * (H // p) * (W // p) * (C * p * p + 1) > GRID_THREADS for B, C, H, W, pp in UNSHUFFLE if pp == p), p


@pytest.mark.parametrize("B,C,H,W,p", UNSHUFFLE)
def test_unshuffle_exact(B, C, H, W, p):
    """the token rows of F.pixel_unshuffle in its (c, i, j) column order, bit for bit, with a has_variance column (ld = K + 1) left zero"""
    g = torch.Generator(device=DEV).manual_seed(B * H + C + p)
    x = torch.randn(B, C, H, W, device=DEV, generator=g)
    K, M = C * p * p, B * (H // p) * (W // p)
    buf, out = _guarded(M * (K + 1))
    got = _native.unet_unshuffle(x, p, ld=K + 1, out=out.view(M, K + 1))
    _assert_written(buf, M * (K + 1))
    want = F.pixel_unshuffle(x, p).permute(0, 2, 3, 1).reshape(M, K)
    assert torch.equal(got[:, :K], want) and (got[:, K] == 0).all()
    assert torch.equal(got, _native.unet_unshuffle(x, p, ld=K + 1)), "two calls differ"


@pytest.mark.parametrize("B,C,H,W,p", UNSHUFFLE)
def test_proj_out_vjp(B, C, H, W, p):
    """U [M, N] (the unshuffled cotangent, N = C p p + 1 with the variance column) times proj_out's weight [N, 128]: bit for bit on
    integers, within N + 1 roundings of the float64 sum of |terms| on normal operands"""
    g = torch.Generator(device=DEV).manual_seed(B * H + C + p + 1)
    N, K, M = C * p * p + 1, 128, B * (H // p) * (W // p)
    for exact in (True, False):
        if exact:
            u = torch.randint(-8, 9, (M, N), device=DEV, generator=g).float()
            wt = torch.randint(-8, 9, (N, K), device=DEV, generator=g).float()
        else:
            u, wt = torch.randn(M, N, device=DEV, generator=g), torch.randn(N, K, device=DEV, generator=g)
        buf, out = _guarded(M * K)
        got = _native.unet_proj_out_vjp(u, wt, out=out.view(M, K))
        _assert_written(buf, M * K)
        assert torch.equal(got, _native.unet_proj_out_vjp(u, wt)), "two calls differ"
        want = u.double() @ wt.double()
        if exact:
            assert torch.equal(got.double(), want)
        else:
            bound = (N + 1) * EPS * (u.double().abs() @ wt.double().abs())
            err = (got.double() - want).abs()
            assert (err <= bound).all(), f"max error {err.max():.3e}, worst excess {(err - bound).max():.3e}"


# ---------------------------------------------------------------------------------------------------------------------------------------
# the mapping network's backward (kdb_unet_mapping_vjp)

def mapping_model(mw, augment, user):
    """a one-level U-Net whose mapping network is mw wide; with the augment wrapper its mapping_cond vector is [aug_cond (9), user]"""
    from k_diffusion.models.image_v1 import ImageDenoiserModelV1
    torch.manual_seed(mw + user + augment)
    inner = ImageDenoiserModelV1(3, mw, [1], [8], [False], mapping_cond_dim=user + (9 if augment else 0)).cuda()
    return inner, inner.engine(augment)


def mapping_inputs(rows, augment, user, with_aug, with_mc, mw):
    g = torch.Generator().manual_seed(rows * 7 + user + mw)
    sigma = torch.exp(torch.randn(rows, generator=g) * 1.5)
    aug = torch.randn(rows, 9, generator=g) * 0.3 if with_aug else None
    mc = torch.randn(rows, user, generator=g) if with_mc else None
    dcond = torch.randn(rows, mw, generator=g)
    if augment:
        v = torch.cat([aug if aug is not None else torch.zeros(rows, 9)] + ([mc] if mc is not None else []), 1)
    else:
        v = mc if mc is not None else torch.zeros(rows, user)
    return sigma, aug, mc, dcond, v


def check_mapping_vjp(inner, eng, sigma, aug, mc, dcond, v):
    """kdb_unet_mapping_vjp stage by stage against float64: each output against torch.func.vjp (or the forward) of the oracle's mapping
    network evaluated at the kernel's own previous outputs, within the fp32 roundings of that stage; v bit for bit"""
    rows, mw = dcond.shape
    mcd = v.shape[1]
    cuda = lambda t: None if t is None else t.to(DEV).contiguous()
    bufs = {k: _guarded(rows * (mcd if k == "v" else mw)) for k in ("h0", "a0", "dz0", "dz1", "dh0", "v") if k != "v" or mcd}
    res = eng.mapping_vjp(cuda(sigma), cuda(dcond), cuda(aug), cuda(mc), out={k: o.view(rows, -1) for k, (_, o) in bufs.items()})
    for k, (buf, o) in bufs.items():
        _assert_written(buf, o.numel())
    again = eng.mapping_vjp(cuda(sigma), cuda(dcond), cuda(aug), cuda(mc))
    assert all(torch.equal(res[k], again[k]) for k in bufs), "two calls differ"
    got = {k: t.cpu().double() for k, t in res.items() if t is not None}
    sd = {k: t.detach().cpu().double() for k, t in inner.state_dict().items()}
    lin = lambda i: (lambda t: t @ sd[f"mapping.{i}.weight"].T + sd[f"mapping.{i}.bias"])
    W0, W1 = sd["mapping.0.weight"].abs(), sd["mapping.2.weight"].abs()
    s64, v64, dc = sigma.double(), v.double(), dcond.double()
    has_mc = mcd > 0 and (eng.cfg.augment_wrapper or mc is not None)
    if mcd:
        assert torch.equal(got["v"], v64 if has_mc else torch.zeros_like(v64))
    # h0 = FourierFeatures(log(sigma) / 4) + mapping_cond Linear (v): the oracle's forward ties h0 and its network to oracle.unet_oracle
    te_arg = 2 * math.pi * (s64.log() / 4)[:, None] @ sd["timestep_embed.weight"].T
    h0 = torch.cat([te_arg.cos(), te_arg.sin()], 1) + (v64 @ sd["mapping_cond.weight"].T if has_mc else 0)
    net = lambda h: F.gelu(lin(2)(F.gelu(lin(0)(h))))
    assert torch.allclose(net(h0), U.mapping(sd, s64, v64 if has_mc else None), rtol=1e-12, atol=1e-12)
    b = 8 * EPS * (te_arg.abs().repeat(1, 2) + 1) + ((mcd + 2) * EPS * (v64.abs() @ sd["mapping_cond.weight"].abs().T) if has_mc else 0)
    stages = {"h0": (h0, b)}
    z0 = lin(0)(got["h0"])
    bz0 = (mw + 2) * EPS * (got["h0"].abs() @ W0.T + sd["mapping.0.bias"].abs())
    stages["a0"] = (F.gelu(z0), 1.13 * bz0 + 4 * EPS * (1 + z0.abs()))
    z1 = lin(2)(got["a0"])
    bz1 = (mw + 2) * EPS * (got["a0"].abs() @ W1.T + sd["mapping.2.bias"].abs())
    stages["dz1"] = (torch.func.vjp(F.gelu, z1)[1](dc)[0], dc.abs() * (0.8 * bz1 + 8 * EPS * (1 + z1.abs())))
    s = torch.func.vjp(lin(2), got["a0"])[1](got["dz1"])[0]
    stages["dz0"] = (torch.func.vjp(F.gelu, z0)[1](s)[0],
                     s.abs() * (0.8 * bz0 + 8 * EPS * (1 + z0.abs())) + 1.13 * (mw + 1) * EPS * (got["dz1"].abs() @ W1))
    stages["dh0"] = (torch.func.vjp(lin(0), got["h0"])[1](got["dz0"])[0], (mw + 1) * EPS * (got["dz0"].abs() @ W0))
    for k, (want, bound) in stages.items():
        err = (got[k] - want).abs()
        assert (err <= bound).all(), f"{k}: max error {err.max():.3e}, worst excess {(err - bound).max():.3e}"
    # and the whole backward at once: dh0 against torch.func.vjp of the oracle's network from h0
    want = torch.func.vjp(net, h0)[1](dc)[0]
    assert (got["dh0"] - want).norm() <= 1e-5 * want.norm()


# (augment wrapper, user mapping_cond_dim, aug_cond given, mapping_cond given, mapping_out)
MAPPING = [(True, 0, True, False, 64), (True, 0, False, False, 72), (True, 5, True, True, 256), (False, 6, False, True, 64),
           (False, 6, False, False, 72), (False, 0, False, False, 256)]


@pytest.mark.parametrize("augment,user,with_aug,with_mc,mw", MAPPING)
@pytest.mark.parametrize("rows", [1, 64])
def test_mapping_vjp_against_float64(augment, user, with_aug, with_mc, mw, rows):
    inner, eng = mapping_model(mw, augment, user)
    check_mapping_vjp(inner, eng, *mapping_inputs(rows, augment, user, with_aug, with_mc, mw))


@pytest.mark.parametrize("augment,widest", [(False, 2048), (True, 2046)])
def test_mapping_vjp_shared_memory_edge(augment, widest):
    """(6 mapping_out + mapping_cond_dim) floats of shared memory, at most 48 KiB: the widest mapping network runs and matches, the next even
    width (which the forward still samples) returns KDB_ERR_UNSUPPORTED and launches nothing"""
    mcd = 9 if augment else 0
    assert 6 * widest + mcd <= 12288 < 6 * (widest + 2) + mcd
    inner, eng = mapping_model(widest, augment, 0)
    check_mapping_vjp(inner, eng, *mapping_inputs(2, augment, 0, augment, False, widest))
    inner, eng = mapping_model(widest + 2, augment, 0)
    sigma, dcond = torch.ones(2, device=DEV), torch.zeros(2, widest + 2, device=DEV)
    assert eng.conditioning(sigma).shape[0] == 2
    outs = [torch.zeros(2, widest + 2, device=DEV) for _ in range(5)] + [torch.zeros(2, max(mcd, 1), device=DEV)]
    L, p = _native.lib(), _native.ptr
    torch.cuda.synchronize()
    n0 = _native.launch_count()
    rc = L.kdb_unet_mapping_vjp(eng._h, 2, p(sigma), None, None, p(dcond), *(p(o) for o in outs), _native.stream())
    assert rc == -2 and b"too wide" in L.kdb_last_error(), (rc, L.kdb_last_error())
    assert _native.launch_count() == n0
