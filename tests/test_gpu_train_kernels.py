"""The fp32 training reductions on the H100, kernel by kernel (kdb_wgrad, kdb_wgrad_patch_in / _patch_out, kdb_norm_scale_grad, kdb_colsum,
kdb_split_fac_grad, kdb_class_emb_grad, kdb_denoiser_loss) against float64 sums of the same terms, at the shapes where the kernels branch:
ragged last row chunks, per-image chunks that are neither full nor alone, the grid-stride loop, strided operands and per-image outputs.

Two kinds of operands.  Exact ones (small integers, powers of two for scale and rstd) make every partial sum exact in fp32, so the kernel
must equal the float64 sum bit for bit whatever its summation order: a dropped, doubled or misplaced row, column, chunk or image fails.
Random normal ones hold each element to the fp32 accumulation bound over the float64 sum of |terms|.  Every output starts as NaN with a
sentinel after it (unwritten elements and writes past the end both show), and two calls must give the same bits."""
import ctypes
import math
import zlib

import pytest
import torch

from k_diffusion import _native

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                 # fp32 unit roundoff
SENTINEL = 7.0
NUM_SMS, TILE = 132, 64        # the H100's SMs, wgrad_kernel's output tile
PART_FLOATS = 1 << 22          # kTrainPartFloats: the partials scratch of every reduction


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def _ints(shape, g, lo=-4, hi=4):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g, dtype=torch.int32).float()


def _guarded(n, pad=64):
    """(buffer, view): n NaN floats to be written followed by `pad` sentinel floats"""
    buf = torch.full((n + pad,), float("nan"), device="cuda")
    buf[n:] = SENTINEL
    return buf, buf[:n]


def _assert_written(buf, n):
    assert not buf[:n].isnan().any(), "an output element was left unwritten"
    assert (buf[n:] == SENTINEL).all(), "a write past the end of the output"


def _assert_exact(got, want):
    got = got.double().cpu()
    bad = got != want
    assert not bad.any(), (f"{int(bad.sum())} elements differ from the exact sum, first at {bad.nonzero()[0].tolist()}: "
                           f"{got[bad][:4]} vs {want[bad][:4]}")


def _assert_bounded(got, want, bound):
    err = (got.double().cpu() - want).abs()
    assert (err <= bound).all(), f"max error {err.max():.3e}, worst excess {(err - bound).max():.3e}"


def _chunks(M, N, K):
    """wgrad_chunk: the row chunks of the weight-gradient reduction, -> (chunk, count, last chunk's rows)"""
    tiles = math.ceil(N / TILE) * math.ceil(K / TILE)
    chunks = min(math.ceil(2 * NUM_SMS / tiles), math.ceil(M / 256))
    chunks = max(1, min(chunks, PART_FLOATS // (N * K)))
    chunk = -(-math.ceil(M / chunks) // 16) * 16
    count = math.ceil(M / chunk)
    return chunk, count, M - (count - 1) * chunk


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_wgrad: rows and the TokenMerge gather, fp32 and tf32

WGRAD_M = [1, 15, 16, 17, 255, 256, 257, 1000, 40000]
WGRAD_NK = [(3, 5), (64, 64), (70, 130)]


def test_wgrad_cases_reach_a_short_last_chunk():
    """the M above leave, among others, a last chunk shorter than the rest (wgrad_kernel's rows = M - r0 < chunk)"""
    short = [(M, N, K) for M in WGRAD_M for N, K in WGRAD_NK if _chunks(M, N, K)[1] > 1 and _chunks(M, N, K)[2] < _chunks(M, N, K)[0]]
    assert {M for M, _, _ in short} >= {257, 1000, 40000}, short


def _strided(t, pad_before, pad_after):
    """t [m, n] copied into rows pad_before + n + pad_after floats apart (the rows' neighbours NaN) -> the [m, n] view"""
    wide = torch.full((t.shape[0], pad_before + t.shape[1] + pad_after), float("nan"), device=t.device)
    wide[:, pad_before:pad_before + t.shape[1]] = t
    return wide[:, pad_before:pad_before + t.shape[1]]


def _run_wgrad(dy, x, precision, **kw):
    N, K = dy.shape[1], x.shape[-1] * (4 if kw.get("merge") else 1)
    buf, out = _guarded(N * K)
    got = _native.wgrad(dy, x, precision, out=out.view(N, K), **kw)
    _assert_written(buf, N * K)
    assert torch.equal(got, _native.wgrad(dy, x, precision, **kw)), "two calls differ"
    return got


@pytest.mark.parametrize("precision", [_native.PREC_FP32, _native.PREC_TF32], ids=["fp32", "tf32"])
@pytest.mark.parametrize("N,K", WGRAD_NK)
@pytest.mark.parametrize("M", WGRAD_M)
def test_wgrad_rows_exact(M, N, K, precision):
    """small integers (exact in tf32 too): the float64 sum bit for bit, dy and x with row strides past N and K"""
    g = _gen("wgrad", M, N, K)
    dy, x = _ints((M, N), g), _ints((M, K), g)
    got = _run_wgrad(_strided(dy, 1, 2), _strided(x, 3, 0), precision)
    _assert_exact(got, dy.double().T.cpu() @ x.double().cpu())


@pytest.mark.parametrize("N,K", WGRAD_NK)
@pytest.mark.parametrize("M", WGRAD_M)
def test_wgrad_rows_random_fp32(M, N, K):
    g = _gen("wgrad_rand", M, N, K)
    dy, x = torch.randn(M, N, device="cuda", generator=g), torch.randn(M, K, device="cuda", generator=g)
    got = _run_wgrad(_strided(dy, 0, 5), x, _native.PREC_FP32)
    a, b = dy.double().cpu(), x.double().cpu()
    _assert_bounded(got, a.T @ b, 1.01 * M * U * (a.abs().T @ b.abs()))


def _merge_gather(fine, hc, wc):
    B, Cf = fine.shape[0], fine.shape[-1]
    return fine.view(B, hc, 2, wc, 2, Cf).permute(0, 1, 3, 2, 4, 5).reshape(B * hc * wc, 4 * Cf)   # TokenMerge: (nh nw e)


@pytest.mark.parametrize("precision", [_native.PREC_FP32, _native.PREC_TF32], ids=["fp32", "tf32"])
@pytest.mark.parametrize("B,hc,wc,Cf,N", [(1, 1, 1, 1, 1), (2, 4, 6, 24, 40), (3, 16, 4, 48, 96), (5, 7, 3, 17, 65), (64, 8, 8, 32, 64),
                                           (4, 8, 16, 64, 128)])
def test_wgrad_merge_exact(B, hc, wc, Cf, N, precision):
    """the TokenMerge gather read in place on grids with hc != wc: the plain-rows result on the gathered rows, bit for bit the exact sum"""
    g = _gen("merge", B, hc, wc, Cf, N)
    fine = _ints((B, 2 * hc, 2 * wc, Cf), g)
    M = B * hc * wc
    dy = _ints((M, N), g)
    got = _run_wgrad(_strided(dy, 2, 3), fine, precision, merge=(hc, wc))
    gathered = _merge_gather(fine, hc, wc)
    _assert_exact(got, dy.double().T.cpu() @ gathered.double().cpu())
    assert torch.equal(got, _native.wgrad(dy, gathered, precision))


@pytest.mark.parametrize("B,hc,wc,Cf,N", [(2, 4, 6, 24, 40), (5, 7, 3, 17, 65), (64, 8, 8, 32, 64)])
def test_wgrad_merge_random_fp32(B, hc, wc, Cf, N):
    g = _gen("merge_rand", B, hc, wc, Cf, N)
    fine = torch.randn(B, 2 * hc, 2 * wc, Cf, device="cuda", generator=g)
    M = B * hc * wc
    dy = torch.randn(M, N, device="cuda", generator=g)
    got = _run_wgrad(dy, fine, _native.PREC_FP32, merge=(hc, wc))
    a, b = dy.double().cpu(), _merge_gather(fine, hc, wc).double().cpu()
    _assert_bounded(got, a.T @ b, 1.01 * M * U * (a.abs().T @ b.abs()))
    assert torch.equal(got, _native.wgrad(dy, _merge_gather(fine, hc, wc), _native.PREC_FP32))


# ---------------------------------------------------------------------------------------------------------------------------------------
# patch_in and patch_out

def _patch_rows(img, ph, pw):
    """the patch rows [B T, (nh nw c)] of an NCHW image"""
    B, C, H, W = img.shape
    return img.view(B, C, H // ph, ph, W // pw, pw).permute(0, 2, 4, 3, 5, 1).reshape(B * (H // ph) * (W // pw), ph * pw * C)


# (B, C, H, W, ph, pw, N or C0): MNIST's patch 4 on its 7x7 grid, patch 1, non-square patches, H != W, C = 1 and 3, many rows
PATCHES = [(2, 1, 28, 28, 4, 4, 256), (3, 3, 32, 16, 2, 2, 64), (1, 3, 8, 12, 1, 1, 70), (5, 1, 12, 20, 4, 2, 33), (2, 3, 12, 8, 2, 4, 17),
           (40, 3, 40, 24, 2, 2, 96), (64, 3, 32, 32, 4, 4, 256)]


@pytest.mark.parametrize("B,C,H,W,ph,pw,N", PATCHES)
def test_wgrad_patch_in(B, C, H, W, ph, pw, N):
    g = _gen("patch_in", B, C, H, W, ph, pw, N)
    M, K = B * (H // ph) * (W // pw), ph * pw * C
    for exact in (True, False):
        x = _ints((B, C, H, W), g) if exact else torch.randn(B, C, H, W, device="cuda", generator=g)
        dtok = _ints((M, N), g) if exact else torch.randn(M, N, device="cuda", generator=g)
        buf, out = _guarded(N * K)
        got = _native.wgrad_patch_in(dtok, x, (ph, pw), out=out.view(N, K))
        _assert_written(buf, N * K)
        assert torch.equal(got, _native.wgrad_patch_in(dtok, x, (ph, pw)))
        a, b = dtok.double().cpu(), _patch_rows(x, ph, pw).double().cpu()
        if exact:
            _assert_exact(got, a.T @ b)
        else:
            _assert_bounded(got, a.T @ b, 1.01 * M * U * (a.abs().T @ b.abs()))


@pytest.mark.parametrize("B,C,H,W,ph,pw,C0", PATCHES)
def test_wgrad_patch_out(B, C, H, W, ph, pw, C0):
    """dY the patch rows of u, X the out-normed tokens x * (scale * rstd): with scale and rstd powers of two the products stay exact"""
    g = _gen("patch_out", B, C, H, W, ph, pw, C0)
    M, K = B * (H // ph) * (W // pw), ph * pw * C
    for exact in (True, False):
        if exact:
            u, tok = _ints((B, C, H, W), g), _ints((M, C0), g)
            scale = torch.randint(-3, 3, (C0,), device="cuda", generator=g).float().exp2() * (torch.randint(0, 2, (C0,), device="cuda",
                                                                                                              generator=g) * 2 - 1)
            rstd = torch.randint(-4, 2, (M,), device="cuda", generator=g).float().exp2()
        else:
            u, tok = torch.randn(B, C, H, W, device="cuda", generator=g), torch.randn(M, C0, device="cuda", generator=g)
            scale = torch.randn(C0, device="cuda", generator=g)
            rstd = torch.rand(M, device="cuda", generator=g) + 0.5
        buf, out = _guarded(K * C0)
        got = _native.wgrad_patch_out(u, tok, scale, rstd, (ph, pw), out=out.view(K, C0))
        _assert_written(buf, K * C0)
        assert torch.equal(got, _native.wgrad_patch_out(u, tok, scale, rstd, (ph, pw)))
        a = _patch_rows(u, ph, pw).double().cpu()
        b = tok.double().cpu() * scale.double().cpu() * rstd.double().cpu()[:, None]
        if exact:
            _assert_exact(got, a.T @ b)
        else:   # x (scale rstd): two roundings per term before the sum
            _assert_bounded(got, a.T @ b, 1.01 * (M + 2) * U * (a.abs().T @ b.abs()))


# ---------------------------------------------------------------------------------------------------------------------------------------
# norm_scale_grad: the per-image RMSNorm scale gradient

def _unit_rows(rows, C, g):
    """x rows of one magnitude a in {8, 16, 32, 64} with random signs: mean(x^2) = a^2 exactly (+1e-6 rounds away), so rstd = 1 / a and
    x rstd = +-1 exactly"""
    a = torch.randint(3, 7, (rows, 1), device="cuda", generator=g).float().exp2()
    sign = torch.randint(0, 2, (rows, C), device="cuda", generator=g, dtype=torch.int8).float() * 2 - 1
    return a * sign, sign


def _norm_terms(x, dy):
    """float64 dy x rstd per element, rstd = rsqrt(mean(x^2) + 1e-6)"""
    x, dy = x.double().cpu(), dy.double().cpu()
    return dy * x * torch.rsqrt((x * x).mean(1, keepdim=True) + 1e-6)


# (rows per image, images, channels): 1, 49 (7x7), 63, 64, 65, 196 (14x14) and 4096 rows; B up to 128; C of 32, 100, 256 and 513
NORM_CASES = [(1, 128, 32), (49, 8, 100), (63, 3, 513), (64, 5, 256), (65, 4, 32), (196, 16, 256), (4096, 2, 100), (65, 128, 513),
              (196, 128, 32), (4096, 1, 513)]


@pytest.mark.parametrize("R,B,C", NORM_CASES)
def test_norm_scale_grad(R, B, C):
    """per image into a strided output (ldo > C, as the engine's ada_total layout; the gaps stay untouched), x and dy with row strides past
    C; then one sum over all rows"""
    g = _gen("norm", R, B, C)
    rows, ldo, off = R * B, C + 37, 5
    for exact in (True, False):
        if exact:
            x, sign = _unit_rows(rows, C, g)
            dy = _ints((rows, C), g, -8, 8)
            want = (dy * sign).double().cpu().view(B, R, C).sum(1)
        else:
            x, dy = torch.randn(rows, C, device="cuda", generator=g), torch.randn(rows, C, device="cuda", generator=g)
            terms = _norm_terms(x, dy).view(B, R, C)
            want = terms.sum(1)
            # the chunk sums and the chunk-order sum (R + 2 roundings at most), x rstd, and rstd's own error: sum(x^2) over C, the mean,
            # eps and rsqrtf (2 ulp), halved by the square root
            bound = 1.05 * U * (R + 3 + C / 2 + 6) * terms.abs().sum(1)
        xs, dys = _strided(x, 2, 1), _strided(dy, 0, 3)
        n = off + (B - 1) * ldo + C
        buf, flat = _guarded(n)
        _native.norm_scale_grad(xs, dys, R, out=flat[off:], ldo=ldo)
        assert (buf[n:] == SENTINEL).all(), "a write past the end of the output"
        got = flat[off:].unfold(0, C, ldo) if B > 1 else flat[off:off + C].view(1, C)
        written = torch.zeros(n, dtype=torch.bool, device="cuda")
        for b in range(B):
            written[off + b * ldo:off + b * ldo + C] = True
        assert not got.isnan().any() and buf[:n][~written].isnan().all(), "unwritten channels, or writes between the images"
        assert torch.equal(got, _native.norm_scale_grad(xs, dys, R)), "two calls differ (or the strided output differs)"
        if exact:
            _assert_exact(got, want)
        else:
            _assert_bounded(got, want, bound)
        # all rows as one image (out_norm and the mapping network's norms: ldo unused)
        buf1, out1 = _guarded(C)
        whole = _native.norm_scale_grad(xs, dys, out=out1)
        _assert_written(buf1, C)
        if exact:
            _assert_exact(whole.view(1, C), want.sum(0, keepdim=True))
        else:
            _assert_bounded(whole.view(1, C), want.sum(0, keepdim=True), 1.05 * U * (rows + 3 + C / 2 + 6) * terms.abs().sum((0, 1))[None])


# ---------------------------------------------------------------------------------------------------------------------------------------
# colsum

@pytest.mark.parametrize("C", [1, 3, 8, 16])
@pytest.mark.parametrize("rows", [1, 255, 256, 257, 511, 512, 513, 10241, 100000])
def test_colsum(rows, C):
    g = _gen("colsum", rows, C)
    for exact in (True, False):
        p = _ints((rows, C), g) if exact else torch.randn(rows, C, device="cuda", generator=g)
        buf, out = _guarded(C)
        got = _native.colsum(p, out=out)
        _assert_written(buf, C)
        assert torch.equal(got, _native.colsum(p))
        want = p.double().cpu().sum(0)
        if exact:
            _assert_exact(got, want)
        else:
            _assert_bounded(got, want, 1.01 * rows * U * p.double().cpu().abs().sum(0))


# ---------------------------------------------------------------------------------------------------------------------------------------
# split_fac: one sum over B H W C elements, grid-striding past 132 x 16 blocks of 256 threads

SPLIT_STRIDE = NUM_SMS * 16 * 256   # 540,672 elements in the first pass of the grid


# (B, H, W, C): under, at and just over one pass of the grid (12 elements on a second trip), and many passes
@pytest.mark.parametrize("B,H,W,C", [(2, 6, 10, 7), (1, 2, 2, 135167), (1, 32, 32, 528), (3, 2, 2, 45057), (16, 16, 16, 256), (4, 32, 32, 256)])
def test_split_fac_grad(B, H, W, C):
    total = B * H * W * C
    assert total != SPLIT_STRIDE or (B, H, W, C) == (1, 32, 32, 528)
    g = _gen("split", B, H, W, C)
    for exact in (True, False):
        if exact:   # entries in {-1, 0, 1}: every partial is an integer below 2^24
            y, skip, dup = (_ints(s, g, -1, 1) for s in ((B, H // 2, W // 2, 4 * C), (B, H, W, C), (B, H, W, C)))
        else:
            y, skip, dup = (torch.randn(s, device="cuda", generator=g) for s in ((B, H // 2, W // 2, 4 * C), (B, H, W, C), (B, H, W, C)))
        buf, out = _guarded(1)
        got = _native.split_fac_grad(y, skip, dup, out=out)
        _assert_written(buf, 1)
        assert torch.equal(got, _native.split_fac_grad(y, skip, dup))
        yf = y.view(B, H // 2, W // 2, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, C)   # TokenSplit: coarse (nh nw e) -> fine
        terms = (yf.double() - skip.double()) * dup.double()
        want = terms.sum().cpu().view(1)
        if exact:
            _assert_exact(got, want)
        else:   # y - skip, the product, the per-thread sums, the block sum and the sum over blocks
            _assert_bounded(got, want, 1.01 * (total + 2) * U * terms.abs().sum().cpu())


# ---------------------------------------------------------------------------------------------------------------------------------------
# class_emb

@pytest.mark.parametrize("rows,mw,ldd", [(1, 64, 64), (4, 64, 96), (256, 256, 256), (256, 257, 300), (37, 1000, 1000)])
def test_class_emb_grad(rows, mw, ldd):
    """11 rows of class_emb (10 classes and the cond-dropout class 10): a repeated class, absent classes and the dropout class"""
    n_classes = 11
    g = _gen("class_emb", rows, mw, ldd)
    if rows == 1:
        cls = torch.tensor([10], device="cuda")
    else:
        cls = torch.randint(0, 4, (rows,), device="cuda", generator=g) * 3 + 1   # classes 1, 4, 7, 10: repeats and absences
        cls[0] = 10
    for exact in (True, False):
        demb = _ints((rows, mw), g) if exact else torch.randn(rows, mw, device="cuda", generator=g)
        demb_s = _strided(demb, 0, ldd - mw) if ldd > mw else demb
        buf, out = _guarded(n_classes * mw)
        got = _native.class_emb_grad(demb_s, cls, n_classes, out=out.view(n_classes, mw))
        _assert_written(buf, n_classes * mw)
        assert torch.equal(got, _native.class_emb_grad(demb_s, cls, n_classes))
        onehot = torch.nn.functional.one_hot(cls.cpu(), n_classes).double()
        want = onehot.T @ demb.double().cpu()
        absent = onehot.sum(0) == 0
        assert (got.cpu()[absent] == 0).all() and absent.any()
        if exact:
            _assert_exact(got, want)
        else:
            _assert_bounded(got, want, 1.01 * rows * U * (onehot.T @ demb.double().cpu().abs()))


# ---------------------------------------------------------------------------------------------------------------------------------------
# The partials scratch limits: just within them a reduction works and matches, one chunk over it is refused before any launch

def _refused(fn, out):
    before, snapshot = _native.launch_count(), out.clone()
    with pytest.raises(RuntimeError, match="-4"):   # KDB_ERR_BAD_SHAPE
        fn()
    torch.cuda.synchronize()
    assert _native.launch_count() == before and torch.equal(out.isnan(), snapshot.isnan())


def test_norm_scale_grad_at_the_partials_limit():
    """one image of C = 1024 channels: ceil(rows / 64) C <= 2^22 allows 262,144 rows; 262,145 rows need one chunk more"""
    C = 1024
    rows = PART_FLOATS // C * 64
    g = _gen("norm_limit")
    x, sign = _unit_rows(rows + 1, C, g)
    dy = _ints((rows + 1, C), g, -8, 8)
    want = (dy[:rows] * sign[:rows]).sum(0, dtype=torch.float64).cpu()
    del sign
    buf, out = _guarded(C)
    got = _native.norm_scale_grad(x[:rows], dy[:rows], out=out)
    _assert_written(buf, C)
    _assert_exact(got, want)
    buf2, out2 = _guarded(C)
    _refused(lambda: _native.norm_scale_grad(x, dy, out=out2), out2)
    assert out2.isnan().all()
    del x, dy
    torch.cuda.empty_cache()


def test_colsum_at_the_partials_limit():
    """C = 1024 columns: ceil(rows / 256) C <= 2^22 allows 1,048,576 rows; one row more needs one chunk more"""
    C = 1024
    rows = PART_FLOATS // C * 256
    g = _gen("colsum_limit")
    p = torch.randint(-4, 5, (rows + 1, C), device="cuda", generator=g, dtype=torch.int8).float()
    want = p[:rows].sum(0, dtype=torch.float64).cpu()
    buf, out = _guarded(C)
    got = _native.colsum(p[:rows], out=out)
    _assert_written(buf, C)
    _assert_exact(got, want)
    buf2, out2 = _guarded(C)
    _refused(lambda: _native.colsum(p, out=out2), out2)
    assert out2.isnan().all()
    del p
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------------------------
# kdb_denoiser_loss: Denoiser (karras, soft-min-snr and snr weights) and SimpleLossDenoiser

def _loss_reference(kind, x, noise, sigma, w, sd):
    """the reference's formula (layers.py:76-86 with scales == 1, :107-111) in x's dtype on the CPU, -> (loss, d loss / d f) of a given f"""
    def run(f):
        s = sigma.view(-1, *[1] * (x.ndim - 1))
        var = s ** 2 + sd ** 2
        c_skip, c_out = sd ** 2 / var, s * sd / var ** 0.5
        noised = x + noise * s
        f = f.detach().requires_grad_(True)
        if kind == _native.LOSS_DENOISER:
            loss = ((f - (x - c_skip * noised) / c_out) ** 2).flatten(1).mean(1) * w
        else:
            loss = (((noised - (f * c_out + noised * c_skip)) / s - noise) ** 2).flatten(1).mean(1)
        loss.sum().backward()
        return loss.detach(), f.grad
    return run


WEIGHTINGS = {"karras": lambda s, sd: torch.ones_like(s), "soft-min-snr": lambda s, sd: (s * sd) ** 2 / (s ** 2 + sd ** 2) ** 2,
              "snr": lambda s, sd: sd ** 2 / (s ** 2 + sd ** 2)}


@pytest.mark.parametrize("weighting", ["karras", "soft-min-snr", "snr", "simple"])
@pytest.mark.parametrize("n,B", [(1, 128), (255, 7), (256, 3), (257, 128), (784, 16), (3072, 5)])
def test_denoiser_loss_against_float64(n, B, weighting):
    """sigma log-uniform over [1e-3, 1e3]; loss and cotangent within 8x the distance of torch's fp32 evaluation of the formula from float64
    (plus a few units of roundoff); a NULL cotangent leaves the loss's bits unchanged"""
    g = torch.Generator().manual_seed(n * 1000 + B + len(weighting))
    sd = 0.5 if weighting != "snr" else 1.0
    x = torch.randn(B, n, generator=g) * 0.5
    noise = torch.randn(B, n, generator=g)
    sigma = torch.exp(torch.rand(B, generator=g) * (2 * math.log(1e3)) - math.log(1e3))
    sigma[0], sigma[-1] = 1e-3, 1e3
    f = torch.randn(B, n, generator=g)
    kind = _native.LOSS_SIMPLE if weighting == "simple" else _native.LOSS_DENOISER
    w = WEIGHTINGS.get(weighting, WEIGHTINGS["karras"])(sigma, sd)
    loss, cot = _native.denoiser_loss(x.cuda(), noise.cuda(), sigma.cuda(), w.cuda(), sd, f.cuda(), kind)
    l64, c64 = _loss_reference(kind, x.double(), noise.double(), sigma.double(), w.double(), sd)(f.double())
    l32, c32 = _loss_reference(kind, x, noise, sigma, w, sd)(f)
    loss, cot = loss.cpu().double(), cot.cpu().double()
    assert ((loss - l64).abs() <= 8 * (l32.double() - l64).abs() + 8 * U * l64.abs()).all(), (loss, l64, l32)
    err = (cot - c64).norm(dim=1)
    ref = (c32.double() - c64).norm(dim=1)
    assert (err <= 8 * ref + 8 * U * c64.norm(dim=1)).all(), (err / c64.norm(dim=1)).max()
    # no cotangent: the loss alone, the same bits
    xs, ns, ss, ws, fs = (t.cuda() for t in (x, noise, sigma, w, f))
    alone = torch.full((B,), float("nan"), device="cuda")
    L = _native.lib()
    _native.check(L.kdb_denoiser_loss(kind, _native.ptr(xs), _native.ptr(ns), _native.ptr(ss), _native.ptr(ws), ctypes.c_float(sd),
                                      _native.ptr(fs), _native.ptr(alone), None, B, n, _native.stream()))
    assert torch.equal(alone.cpu().double(), loss)
