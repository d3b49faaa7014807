"""KID / FID on the H100: the native MMD sums, kernel matrix, mean / covariance, kid and fid against the float64 oracle at the fixture
shapes, edge sizes and one full 5000 x 5000 x 2048 kid partition; determinism, launch counts, refusals."""
import json

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz
from oracle import metrics_oracle as O

pytestmark = pytest.mark.gpu

META = json.loads((GOLDEN / "metrics_meta.json").read_text())
CASES = sorted(META["cases"])
F32 = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def arrays():
    return load_npz("metrics.npz")


def _kid_tol(x, y, max_size, ref_err=None):
    """1e-6 of |term_1| + |term_2| + |term_3| (the largest over the partitions); with the reference's recorded error, that error or a
    quarter fp32 ulp of the terms' magnitude, whichever is larger (one recorded error is one draw, and can fall below what rounding
    each fp32 kernel value alone gives)."""
    terms = O.kid_terms(x, y, max_size)
    mag = max(abs(sxx) / (len(x) * (len(x) - 1)) + abs(syy) / (len(y) * (len(y) - 1)) + 2 * abs(sxy) / (len(x) * len(y))
              for sxx, syy, sxy, _ in terms)
    tol = 1e-6 * mag
    return tol if ref_err is None else min(tol, max(ref_err, F32 * mag / 4))


@pytest.mark.parametrize("name", CASES)
def test_fixture_shapes_against_the_oracle(arrays, name):
    import k_diffusion as K
    E = K.evaluation
    rec = META["cases"][name]
    x, y = arrays[f"{name}.x"].cuda(), arrays[f"{name}.y"].cuda()
    x64, y64 = x.double().cpu().numpy(), y.double().cpu().numpy()
    ok = O.polynomial_kernel(x64, y64)
    got = E.polynomial_kernel(x, y).double().cpu().numpy()
    # the dot product is one fmaf per k in index order, the reference's a blocked BLAS sum: at d = 2048 the in-order sum's rounding
    # can exceed the recorded error of the reference, never 4 fp32 ulps of the largest element
    assert np.abs(got - ok).max() / np.abs(ok).max() <= max(rec["kernel_err"], 4 * F32)
    sums = K._native.mmd_sums(x, y, [0, len(x)], [0, len(y)]).cpu().numpy()[0]
    terms = O.mmd_terms(x64, y64)
    for q, (a, b) in enumerate(((x64, x64), (y64, y64), (x64, y64))):
        assert abs(sums[q] - terms[q]) <= 4 * F32 * np.abs(O.polynomial_kernel(a, b)).sum(), (q, sums[q], terms[q])
    mmd = float(E.squared_mmd(x, y))
    assert abs(mmd - rec["mmd_oracle"]) <= _kid_tol(x64, y64, 10 ** 9, rec["mmd_err"])
    kid = E.kid(x, y, max_size=rec["max_size"])
    assert kid.dtype == torch.float32 and kid.ndim == 0
    assert abs(float(kid) - rec["kid_oracle"]) <= _kid_tol(x64, y64, rec["max_size"], rec["kid_err"])
    mu, cov = K._native.feature_mean_cov(x)
    mu64, cov64 = O.mean_cov(x64)
    assert np.abs(mu.double().cpu().numpy() - mu64).max() <= max(rec["mean_err"], F32) * np.abs(mu64).max()
    assert np.abs(cov.double().cpu().numpy() - cov64).max() <= max(rec["cov_err"], 2 * F32) * np.abs(cov64).max()
    assert torch.equal(cov, cov.T)
    f = E.fid(x, y)
    assert f.dtype == torch.float32 and f.ndim == 0
    # the eigensolvers differ (cuSOLVER here, LAPACK for the reference): hold fid to the reference's own error, with room for that
    tol = 2 * rec["fid_err"] if "fid_err" in rec else 1e-5 * abs(rec["fid_oracle"])
    assert abs(float(f) - rec["fid_oracle"]) <= max(tol, 1e-5 * abs(rec["fid_oracle"])), (float(f), rec["fid_oracle"])


@pytest.mark.parametrize("m, n, d", [(2, 2, 3), (2, 5, 16), (65, 129, 33), (64, 64, 64), (129, 65, 2049), (300, 257, 130)])
def test_edge_sizes(m, n, d):
    import k_diffusion as K
    g = torch.Generator().manual_seed(m * 1000 + n + d)
    x, y = torch.randn(m, d, generator=g), torch.randn(n, d, generator=g) * 1.1
    x64, y64 = x.double().numpy(), y.double().numpy()
    xc, yc = x.cuda(), y.cuda()
    ok = O.polynomial_kernel(x64, y64)
    assert np.abs(K.evaluation.polynomial_kernel(xc, yc).double().cpu().numpy() - ok).max() <= 1e-6 * np.abs(ok).max()
    assert abs(float(K.evaluation.squared_mmd(xc, yc)) - O.squared_mmd(x64, y64)) <= _kid_tol(x64, y64, 10 ** 9)
    mu, cov = K._native.feature_mean_cov(xc)
    mu64, cov64 = O.mean_cov(x64)
    assert np.abs(mu.double().cpu().numpy() - mu64).max() <= 2 * F32 * np.abs(x64).max()
    assert np.abs(cov.double().cpu().numpy() - cov64).max() <= 1e-6 * np.abs(cov64).max()


def test_unaligned_rows_take_the_scalar_loads():
    """a row slice that starts off a 16-byte boundary (and d not a multiple of 4) reads element by element"""
    import k_diffusion as K
    g = torch.Generator().manual_seed(5)
    base = torch.randn(101, 8, generator=g).cuda()
    x = base.view(-1)[1:1 + 100 * 8].view(100, 8)
    assert x.data_ptr() % 16 != 0
    ok = O.mean_cov(x.double().cpu().numpy())[1]
    assert np.abs(K._native.feature_mean_cov(x)[1].double().cpu().numpy() - ok).max() <= 1e-6 * np.abs(ok).max()
    ok = O.squared_mmd(x.double().cpu().numpy(), base.double().cpu().numpy())
    assert abs(float(K.evaluation.squared_mmd(x, base)) - ok) <= _kid_tol(x.double().cpu().numpy(), base.double().cpu().numpy(), 10 ** 9)


def test_full_kid_partition_and_determinism():
    """one 5000 x 5000 x 2048 partition (the size kid runs 10 of at 50 000 samples) against float64; two calls return the same bits"""
    import k_diffusion as K
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(5000, 2048, device="cuda", generator=g).abs_()
    y = torch.randn(5000, 2048, device="cuda", generator=g).abs_() * 1.01
    a, b = K.evaluation.kid(x, y), K.evaluation.kid(x, y)
    assert torch.equal(a.view(1).view(torch.int32), b.view(1).view(torch.int32))
    x64, y64 = x.double(), y.double()     # the float64 oracle's formulas on the GPU (numpy would take minutes here)
    sxx = ((x64 @ x64.T / 2048 + 1) ** 3).sum() - ((x64 * x64).sum(1) / 2048 + 1).pow(3).sum()
    syy = ((y64 @ y64.T / 2048 + 1) ** 3).sum() - ((y64 * y64).sum(1) / 2048 + 1).pow(3).sum()
    sxy = ((x64 @ y64.T / 2048 + 1) ** 3).sum()
    t1, t2, t3 = float(sxx) / 5000 / 4999, float(syy) / 5000 / 4999, float(sxy) * 2 / 5000 / 5000
    assert abs(float(a) - (t1 + t2 - t3)) <= 1e-6 * (abs(t1) + abs(t2) + abs(t3)), (float(a), t1 + t2 - t3)
    s1, s2 = K._native.mmd_sums(x, y, [0, 5000], [0, 5000]), K._native.mmd_sums(x, y, [0, 5000], [0, 5000])
    assert torch.equal(s1, s2)
    f1, f2 = K.evaluation.fid(x[:3000, :512], y[:3000, :512]), K.evaluation.fid(x[:3000, :512], y[:3000, :512])
    assert torch.equal(f1, f2)


def test_kid_launch_count_does_not_depend_on_partitions():
    import k_diffusion as K
    g = torch.Generator(device="cuda").manual_seed(3)
    counts = []
    for m, n in ((5000, 5000), (12001, 10001)):
        x, y = torch.randn(m, 64, device="cuda", generator=g), torch.randn(n, 64, device="cuda", generator=g)
        n0 = K._native.launch_count()
        K.evaluation.kid(x, y)
        counts.append(K._native.launch_count() - n0)
    assert counts[0] == counts[1] == 2


def test_kid_of_three_partitions_against_the_oracle():
    import k_diffusion as K
    g = torch.Generator().manual_seed(11)
    x, y = torch.randn(301, 24, generator=g), torch.randn(250, 24, generator=g)
    x64, y64 = x.double().numpy(), y.double().numpy()
    got = float(K.evaluation.kid(x.cuda(), y.cuda(), max_size=100))
    assert abs(got - O.kid(x64, y64, 100)) <= _kid_tol(x64, y64, 100)


def test_batched_squared_mmd_is_one_call_per_batch():
    import k_diffusion as K
    g = torch.Generator().manual_seed(12)
    x, y = torch.randn(3, 2, 40, 9, generator=g), torch.randn(3, 2, 31, 9, generator=g)
    n0 = K._native.launch_count()
    got = K.evaluation.squared_mmd(x.cuda(), y.cuda())
    assert K._native.launch_count() - n0 == 2 and got.shape == (3, 2) and got.dtype == torch.float32
    want = O.squared_mmd(x.double().numpy(), y.double().numpy())
    assert np.abs(got.double().cpu().numpy() - want).max() <= 1e-5 * np.abs(want).max() + 1e-7
    k = K.evaluation.polynomial_kernel(x.cuda(), y.cuda())
    assert k.shape == (3, 2, 40, 31)
    ok = O.polynomial_kernel(x.double().numpy(), y.double().numpy())
    assert np.abs(k.double().cpu().numpy() - ok).max() <= 1e-6 * np.abs(ok).max()
    with pytest.raises(ValueError, match="batch"):
        K.evaluation.squared_mmd(x.cuda(), y[:1].cuda())


def test_custom_kernel_goes_through_the_torch_formula():
    import k_diffusion as K
    g = torch.Generator().manual_seed(13)
    x, y = torch.randn(30, 5, generator=g).cuda(), torch.randn(20, 5, generator=g).cuda()
    calls = []

    def rbf(a, b):
        calls.append((a.shape, b.shape))
        return torch.exp(-torch.cdist(a, b) ** 2 / 2)
    n0 = K._native.launch_count()
    got = K.evaluation.squared_mmd(x, y, kernel=rbf)
    assert K._native.launch_count() == n0 and len(calls) == 3
    kxx, kyy, kxy = rbf(x, x).double(), rbf(y, y).double(), rbf(x, y).double()
    want = ((kxx.sum() - kxx.trace()) / 30 / 29 + (kyy.sum() - kyy.trace()) / 20 / 19 - kxy.sum() * 2 / 30 / 20).item()
    assert abs(float(got) - want) <= 1e-5
    # the default kernel passed explicitly is the native call
    n0 = K._native.launch_count()
    K.evaluation.squared_mmd(x, y, kernel=K.evaluation.polynomial_kernel)
    assert K._native.launch_count() - n0 == 2


def test_small_segments_give_nan_as_the_reference():
    import k_diffusion as K
    x, y = torch.randn(1, 6).cuda(), torch.randn(7, 6).cuda()
    assert torch.isnan(K.evaluation.squared_mmd(x, y))
    assert torch.isnan(K.evaluation.kid(torch.randn(3, 6).cuda(), torch.randn(7, 6).cuda(), max_size=2))   # partitions of 1 x row
    assert torch.isfinite(K.evaluation.squared_mmd(torch.randn(2, 6).cuda(), torch.randn(2, 6).cuda()))


def test_dtypes_are_converted_to_fp32():
    import k_diffusion as K
    g = torch.Generator().manual_seed(14)
    x, y = torch.randn(50, 16, generator=g).cuda(), torch.randn(40, 16, generator=g).cuda()
    ref_k, ref_f = K.evaluation.kid(x, y), K.evaluation.fid(x, y)
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        xd, yd = x.to(dt), y.to(dt)
        k, f = K.evaluation.kid(xd, yd), K.evaluation.fid(xd, yd)
        assert k.dtype == f.dtype == torch.float32
        assert torch.equal(k, K.evaluation.kid(xd.float(), yd.float())) and torch.equal(f, K.evaluation.fid(xd.float(), yd.float()))
    assert torch.isfinite(ref_k) and torch.isfinite(ref_f)


def test_same_distribution_scores_near_zero():
    import k_diffusion as K
    g = torch.Generator(device="cuda").manual_seed(15)
    x, y = torch.randn(4000, 64, device="cuda", generator=g), torch.randn(4000, 64, device="cuda", generator=g)
    # fp32 eigh: the two square roots of tr(2 C) ~ 128 round to a few 1e-5 of it, as in the reference on the same card
    assert abs(float(K.evaluation.fid(x, x))) < 1e-4 * 2 * float(torch.cov(x.T).trace())
    assert abs(float(K.evaluation.kid(x, y))) < 1e-3
    assert float(K.evaluation.fid(x, y + 1)) > 60          # the mean term alone is 64


def test_scores_of_sampled_images_through_a_feature_function():
    """sample_images output passed through a feature function (here a fixed random projection) scores like any features"""
    import k_diffusion as K

    class One:
        num_processes, process_index, is_main_process = 1, 0, True

        def gather(self, t):
            return t
    model = lambda x, sigma, **kw: x * 0.5        # noqa: E731
    sigmas = K.sampling.get_sigmas_karras(4, 0.1, 10.0, device="cuda")
    imgs = K.evaluation.sample_images(One(), model, sigmas, 64, 16, (3, 8, 8), 10.0, sampler=K.sampling.sample_euler, seed=1)
    proj = torch.randn(3 * 8 * 8, 32, generator=torch.Generator().manual_seed(0)).cuda()
    feats = imgs.flatten(1) @ proj
    k, f = K.evaluation.kid(feats, feats.flip(0)), K.evaluation.fid(feats, feats.flip(0) * 2)
    assert torch.isfinite(k) and torch.isfinite(f) and float(f) > 0


def test_c_errors_return_before_any_launch():
    import ctypes
    import k_diffusion as K
    L = K._native.lib()
    x = torch.randn(10, 3, device="cuda")
    out = torch.empty(1, 4, dtype=torch.float64, device="cuda")
    xo = (ctypes.c_int64 * 2)(0, 10)
    need = L.kdb_mmd_workspace_bytes(xo, xo, 1)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n0 = K._native.launch_count()
    assert L.kdb_mmd_sums(p(x), 10, p(x), 10, 3, xo, xo, 1, p(out), p(ws), need - 8, s) == -5
    assert L.kdb_mmd_sums(p(x), 9, p(x), 10, 3, xo, xo, 1, p(out), p(ws), need, s) == -4
    assert L.kdb_polynomial_kernel(p(x), p(x), p(x), 1, 10, 10, 0, s) == -4
    assert L.kdb_feature_mean_cov(p(x), 0, 3, p(x), p(x), s) == -4
    assert K._native.launch_count() == n0
    assert L.kdb_mmd_sums(p(x), 10, p(x), 10, 3, xo, xo, 1, p(out), p(ws), need, s) == 0
    assert K._native.launch_count() == n0 + 2
    want = O.mmd_terms(x.double().cpu().numpy(), x.double().cpu().numpy())[3]
    assert float(out[0, 3]) == pytest.approx(want, rel=1e-5, abs=1e-6)
