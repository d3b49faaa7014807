"""KID / FID scoring without a GPU: the float64 oracle against the reference's fixtures, kid's partition bounds, the public signatures,
the refusals of CPU features and unequal batch dimensions, and tf32_mode."""
import json

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_npz
from oracle import metrics_oracle as O

META = json.loads((GOLDEN / "metrics_meta.json").read_text())
CASES = sorted(META["cases"])


@pytest.fixture(scope="module")
def arrays():
    return load_npz("metrics.npz")


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_reference_fixtures(arrays, name):
    """the reference's fp32 results lie within a few fp32 roundings of the float64 oracle (fid at d = 2048 with fewer rows than
    features is ill-conditioned: there the recorded error is the reference's own, and only its magnitude is checked)"""
    rec = META["cases"][name]
    x, y = arrays[f"{name}.x"].double().numpy(), arrays[f"{name}.y"].double().numpy()
    k = O.polynomial_kernel(x, y)
    assert np.abs(arrays[f"{name}.kxy"].double().numpy() - k).max() <= 1e-6 * np.abs(k).max()
    terms = O.mmd_terms(x, y)
    scale = sum(abs(float(t)) for t in terms[:3]) / (len(x) * len(y))
    assert abs(rec["mmd"] - float(terms[3])) <= 1e-5 * scale + 1e-7
    assert rec["mmd_oracle"] == pytest.approx(float(terms[3]), rel=1e-12, abs=1e-15)
    assert rec["kid_oracle"] == pytest.approx(O.kid(x, y, rec["max_size"]), rel=1e-12, abs=1e-15)
    assert abs(rec["kid"] - rec["kid_oracle"]) <= 1e-5 * scale + 1e-7
    assert rec["fid_oracle"] == pytest.approx(O.fid(x, y), rel=1e-9)
    if "fid" in rec and x.shape[0] > x.shape[1]:
        assert abs(rec["fid"] - rec["fid_oracle"]) <= 1e-4 * abs(rec["fid_oracle"]) + 1e-5


@pytest.mark.parametrize("name", CASES)
def test_kid_partition_bounds_are_the_references(name):
    import k_diffusion as K
    rec = META["cases"][name]
    m, n = rec["kid_bounds_x"][-1], rec["kid_bounds_y"][-1]
    P = len(rec["kid_bounds_x"]) - 1
    assert P == -(-max(m, n) // rec["max_size"])
    assert K.evaluation._partition_bounds(m, P) == rec["kid_bounds_x"]
    assert K.evaluation._partition_bounds(n, P) == rec["kid_bounds_y"]
    assert O.partition_bounds(m, P) == rec["kid_bounds_x"]


def test_partition_bounds_round_half_to_even():
    """the ties of the fixtures: 22.5 -> 22, 13.5 -> 14, 2.5 -> 2, 7.5 -> 8, 12.5 -> 12"""
    import k_diffusion as K
    assert META["cases"]["ties2"]["kid_bounds_x"] == [0, 22, 45] and META["cases"]["ties2"]["kid_bounds_y"] == [0, 14, 27]
    assert K.evaluation._partition_bounds(15, 6) == [0, 2, 5, 8, 10, 12, 15]
    assert K.evaluation._partition_bounds(12001, 3) == [0, 4000, 8001, 12001]


def test_signatures_equal_the_references():
    import inspect
    import k_diffusion as K
    for name, want in META["signatures"].items():
        got = [[p, v.kind.name, None if v.default is inspect._empty else repr(v.default)]
               for p, v in inspect.signature(getattr(K.evaluation, name)).parameters.items()]
        if name == "squared_mmd":      # the default is the module's own polynomial_kernel; its repr holds an address
            assert got[2][2].startswith("<function polynomial_kernel") and want[2][2].startswith("<function polynomial_kernel")
            got[2][2] = want[2][2]
        assert got == want, name


@pytest.mark.parametrize("fn", ["polynomial_kernel", "squared_mmd", "kid", "fid"])
def test_cpu_features_are_refused(fn):
    import k_diffusion as K
    x = torch.randn(8, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        getattr(K.evaluation, fn)(x, x)


def test_sqrtm_eig_runs_anywhere_and_matches_the_oracle():
    import k_diffusion as K
    a = torch.randn(6, 6, dtype=torch.float64)
    a = a @ a.T + torch.eye(6, dtype=torch.float64)
    s = K.evaluation.sqrtm_eig(a)
    assert np.allclose(s.numpy(), O.sqrtm_eig(a.numpy()), rtol=1e-12, atol=1e-12)
    assert torch.allclose(s @ s, a, rtol=1e-10, atol=1e-10)
    b = a.clone().requires_grad_(True)       # eigh reads one triangle: perturb through a symmetric parametrisation
    assert torch.autograd.gradcheck(lambda b: K.evaluation.sqrtm_eig((b + b.T) / 2), (b,))
    with pytest.raises(RuntimeError):
        K.evaluation.sqrtm_eig(torch.ones(3))
    with pytest.raises(RuntimeError):
        K.evaluation.sqrtm_eig(torch.ones(2, 3))


def test_mismatched_batch_dimensions_are_refused(monkeypatch):
    """leading dimensions are compared before any kernel runs; CUDA placement is faked so this runs without a GPU"""
    import k_diffusion as K
    monkeypatch.setattr(K._native, "require_cuda", lambda *t: None)
    x, y = torch.randn(2, 5, 3), torch.randn(1, 4, 3)
    for fn in (K.evaluation.squared_mmd, K.evaluation.polynomial_kernel):
        with pytest.raises(ValueError, match="batch"):
            fn(x, y)
    with pytest.raises(ValueError, match="widths"):
        K.evaluation.squared_mmd(torch.randn(5, 3), torch.randn(4, 2))
    with pytest.raises(ValueError):
        K.evaluation.kid(x, x)


@pytest.mark.parametrize("cudnn, matmul", [(True, True), (False, True), (True, False), (False, False)])
def test_tf32_mode_restores_both_flags(cudnn, matmul):
    import k_diffusion as K
    before = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = cudnn, matmul
        with K.utils.tf32_mode(cudnn=not cudnn, matmul=not matmul):
            assert (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) == (not cudnn, not matmul)
        assert (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) == (cudnn, matmul)
        with pytest.raises(KeyError):
            with K.utils.tf32_mode(cudnn=False, matmul=False):
                raise KeyError
        assert (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32) == (cudnn, matmul)
        with K.utils.tf32_mode(matmul=not matmul):        # a flag left as None is not touched
            assert torch.backends.cudnn.allow_tf32 == cudnn
        assert torch.backends.cuda.matmul.allow_tf32 == matmul

        @K.utils.tf32_mode(matmul=False)
        def inner():
            return torch.backends.cuda.matmul.allow_tf32
        assert inner() is False and torch.backends.cuda.matmul.allow_tf32 == matmul
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = before


def test_c_entry_points_refuse_bad_arguments_without_a_gpu():
    """argument and workspace errors come back as KDB_ERR_* before any CUDA call"""
    import ctypes
    from k_diffusion import _native
    L = _native.lib()
    i64 = ctypes.c_int64
    xo, yo = (i64 * 3)(0, 5, 10), (i64 * 3)(0, 4, 8)
    need = L.kdb_mmd_workspace_bytes(xo, yo, 2)
    assert need > 0
    bad = (i64 * 3)(0, 6, 5)                                     # decreasing
    assert L.kdb_mmd_workspace_bytes(bad, yo, 2) == -4
    assert L.kdb_mmd_workspace_bytes(xo, yo, 0) == -1
    p = ctypes.c_void_p(256)                                     # never dereferenced: validation fails first
    assert L.kdb_mmd_sums(p, 10, p, 8, 3, xo, yo, 2, p, p, need - 1, None) == -5
    assert b"workspace" in L.kdb_last_error()
    assert L.kdb_mmd_sums(p, 9, p, 8, 3, xo, yo, 2, p, p, need, None) == -4       # x has 9 rows, the bounds reach 10
    assert L.kdb_mmd_sums(p, 10, p, 8, 0, xo, yo, 2, p, p, need, None) == -4      # d = 0
    assert L.kdb_mmd_sums(None, 10, p, 8, 3, xo, yo, 2, p, p, need, None) == -1
    assert L.kdb_polynomial_kernel(p, p, p, 1, 0, 4, 3, None) == -4
    assert L.kdb_polynomial_kernel(p, p, p, 70000, 4, 4, 3, None) == -4
    assert L.kdb_feature_mean_cov(p, 0, 4, p, p, None) == -4
    assert L.kdb_feature_mean_cov(p, 2 ** 31, 4, p, p, None) == -4
    assert L.kdb_feature_mean_cov(None, 5, 4, p, p, None) == -1
