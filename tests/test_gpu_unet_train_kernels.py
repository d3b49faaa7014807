"""The U-Net's backward kernels one by one against float64 torch.func, at the edges a whole-model tolerance cannot see: the convolution's
weight gradient and (the forward convolution on the flipped weight) input gradient at the zero-padded borders, with one and two sources, ks 1
and 3, on 7x7, 8x8 and odd non-square grids with N not a multiple of 64; the AdaGN (+ GELU) backward with one and several groups and its
mapper-output rows; the resampling adjoints at the reflect borders and their adjointness.  Integer-valued operands, where the arithmetic is
exact, must match bit for bit."""
import pytest
import torch
from torch.nn import functional as F

from oracle import unet_oracle as U

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


def adagn64(x, cond, off, groups, gelu):
    C = x.shape[-1]
    wgt, bias = cond[:, off:off + C], cond[:, off + C:off + 2 * C]
    y = F.group_norm(nchw(x), groups, eps=U.GN_EPS) * (wgt + 1)[:, :, None, None] + bias[:, :, None, None]
    return (F.gelu(y) if gelu else y).permute(0, 2, 3, 1)


@pytest.mark.parametrize("groups,c1,c2", [(1, 24, 0), (3, 48, 0), (2, 32, 32), (4, 64, 64)])
@pytest.mark.parametrize("gelu", [False, True])
def test_adagn_vjp_against_float64(groups, c1, c2, gelu):
    g = torch.Generator().manual_seed(groups * 100 + c1 + c2 + gelu)
    B, h, w, C = 2, 5, 6, c1 + c2
    x = torch.randn(B, h, w, C, generator=g).double() * 2 + 0.5
    stride, off = 2 * C + 12, 8
    cond = torch.randn(B, stride, generator=g).double() * 0.5
    dy = torch.randn(B, h, w, C, generator=g).double()
    add = torch.randn(B, h, w, C, generator=g).double()
    _, pull = torch.func.vjp(lambda xx, cc: adagn64(xx, cc, off, groups, gelu), x, cond)
    dx_want, dc_want = pull(dy)
    f = lambda t: t.float().to(DEV).contiguous()
    x1, x2 = f(x[..., :c1]), (f(x[..., c1:]) if c2 else None)
    dx1, dx2, dss = _native.unet_adagn_vjp(x1, f(dy), f(cond), off, groups, gelu, x2=x2, add=f(add))
    dx = torch.cat([dx1, dx2], -1) if c2 else dx1
    tol = lambda want: 2e-5 * want.abs().max().item() + 1e-6
    assert ((dx.cpu().double() - add) - dx_want).abs().max() <= tol(dx_want)
    got_dc = dss.cpu().double()[:, off:off + 2 * C]
    assert (got_dc - dc_want[:, off:off + 2 * C]).abs().max() <= tol(dc_want)
    assert torch.isnan(dss[:, :off]).all() and torch.isnan(dss[:, off + 2 * C:]).all()   # nothing outside its rows is written
    again = _native.unet_adagn_vjp(x1, f(dy), f(cond), off, groups, gelu, x2=x2, add=f(add))
    assert torch.equal(again[0], dx1) and torch.equal(again[2][:, off:off + 2 * C], dss[:, off:off + 2 * C])


def resample64(x, up):
    return (U.upsample if up else U.downsample)(nchw(x)).permute(0, 2, 3, 1)


@pytest.mark.parametrize("grid", [(2, 2), (7, 7), (8, 8), (5, 9), (6, 10)])
@pytest.mark.parametrize("up", [False, True])
def test_resample_vjp_exact_and_adjoint(grid, up):
    if not up and (grid[0] < 2 or grid[1] < 2):
        pytest.skip("too small")
    g = torch.Generator().manual_seed(grid[0] * 31 + grid[1] + up)
    B, (h, w), C = 2, grid, 6
    x = ints(g, B, h, w, C)
    y0 = resample64(x, up)
    dy = ints(g, *y0.shape)
    _, pull = torch.func.vjp(lambda xx: resample64(xx, up), x)
    (want,) = pull(dy)
    got = _native.unet_resample_vjp(dy.float().to(DEV).contiguous(), h, w, up).cpu().double()
    assert torch.equal(got, want)
    # <resample x, y> = <x, resample^T y>
    assert torch.isclose((y0 * dy).sum(), (x * got).sum(), rtol=0, atol=0)
    add = ints(g, B, h, w, C)
    got_add = _native.unet_resample_vjp(dy.float().to(DEV).contiguous(), h, w, up, add=add.float().to(DEV)).cpu().double()
    assert torch.equal(got_add, want + add)
