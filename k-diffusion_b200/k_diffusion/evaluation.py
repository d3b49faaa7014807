"""Data-parallel sampling driver and sample scoring (reference: k_diffusion/evaluation.py:80-161).

Sampling: every process samples `ceil(n / P)` items in batches, applies `extractor_fn` (identity when the samples themselves are
wanted, sample.py:62) and the per-batch results are gathered across processes -- outside any kernel-timed region, one collective
per batch, as the reference does through `accelerator.gather`.

Scoring: `polynomial_kernel`, `squared_mmd`, `kid`, `sqrtm_eig` and `fid` under the reference's names and signatures, what train.py's
evaluate() calls on the gathered features.  The fp32 products (kernel matrices, MMD sums, feature means and covariances) run on the
native kernels; fid's d x d products and eigendecompositions are torch with TF32 matmul off.  The feature extractors (Inception,
CLIP, DINOv2) are not part of this package: their weights need a download, so `extractor_fn` stays the caller's.

Deviations from the reference, each pinned by a test:
- features must be CUDA tensors; a CPU tensor raises RuntimeError (there is no CPU path);
- float16, bfloat16 and float64 features are converted to fp32, and the scores are fp32 (0-d for kid and fid);
- the leading batch dimensions of x and y must be equal (ValueError), they are not broadcast;
- the MMD sums, and kid's mean over its partitions, are formed in fp64 from fp32 kernel values, and the feature means are fp64 sums:
  at least as accurate as the reference's fp32 sums, not bit-identical to them;
- fid accepts d = 1 (a 1 x 1 covariance), where the reference's torch.cov returns a 0-d tensor and its fid raises IndexError.
A segment (a kid partition or a batch entry) with fewer than 2 rows gives nan, as the reference's 0/0 does.
"""
import math

import torch

from . import _native, parallel, utils

try:
    from tqdm.auto import trange
except ImportError:
    def trange(*args, disable=None):
        return range(*args)


def compute_features(accelerator, sample_fn, extractor_fn, n, batch_size):
    """Same contract as the reference (evaluation.py:80-90).  `accelerator` is anything with `num_processes`, `is_main_process`
    and `gather(tensor)` -- an `accelerate.Accelerator` or `k_diffusion.parallel.ProcessGroup`."""
    n_per_proc = math.ceil(n / accelerator.num_processes)
    feats_all = []
    try:
        for i in trange(0, n_per_proc, batch_size, disable=not accelerator.is_main_process):
            cur_batch_size = min(n - i, batch_size)
            samples = sample_fn(cur_batch_size)[:cur_batch_size]
            feats_all.append(accelerator.gather(extractor_fn(samples)))
    except StopIteration:
        pass
    return torch.cat(feats_all)[:n]


def sample_images(accelerator, model, sigmas, n, batch_size, shape, sigma_max, sampler=None, seed=None, extra_args_fn=None, disable=True):
    """`n` samples of `shape` = (C, H, W) with `sampler(model, x, sigmas, ...)` (default: sample_lms, what sample.py:60 calls).

    seed=None draws the initial latents from torch's global generator on the device like the reference (sample.py:59; results then
    depend on the process layout).  With a seed, latent i is a pure function of (seed, global sample index) (parallel.init_noise),
    so the image set does not depend on how many processes produced it."""
    from . import sampling
    sampler = sampling.sample_lms if sampler is None else sampler
    device = sigmas.device
    P, r = accelerator.num_processes, accelerator.process_index
    done = [0]

    def sample_fn(cur):
        if seed is None:
            x = torch.randn([cur, *shape], device=device) * sigma_max
        else:      # batch k of process r covers the global indices (k * P + r) * batch_size + [0, cur): what gather concatenates
            start = (done[0] * P + r) * batch_size
            x = parallel.init_noise(parallel.sample_seeds(seed, start, start + cur), tuple(shape), sigma_max, device)
        done[0] += 1
        extra = {} if extra_args_fn is None else extra_args_fn(cur)
        return sampler(model, x, sigmas, extra_args=extra, disable=disable)

    return compute_features(accelerator, sample_fn, lambda x: x, n, batch_size)


# ---------------------------------------------------------------------------------------------
# scoring (reference evaluation.py:93-161)
# ---------------------------------------------------------------------------------------------

def _as_features(t, what, ndim=None):
    _native.require_cuda(t)
    if not t.is_floating_point():
        raise TypeError(f"{what}: features must be floating point (got {t.dtype})")
    if t.ndim < 2 or (ndim is not None and t.ndim != ndim):
        raise ValueError(f"{what}: features must be {ndim or 'at least 2'}-D [..., rows, d] (got shape {tuple(t.shape)})")
    return _native.f32c(t)


def _pair(x, y, what, ndim=None):
    x, y = _as_features(x, what, ndim), _as_features(y, what, ndim)
    if x.shape[:-2] != y.shape[:-2]:
        raise ValueError(f"{what}: leading batch dimensions {tuple(x.shape[:-2])} and {tuple(y.shape[:-2])} differ (they are not broadcast)")
    if x.shape[-1] != y.shape[-1] or x.shape[-1] == 0:
        raise ValueError(f"{what}: feature widths {x.shape[-1]} and {y.shape[-1]}")
    return x, y


def polynomial_kernel(x, y):
    """k(x, y) = (x y^T / d + 1)^3 for x [..., m, d] and y [..., n, d] -> [..., m, n] fp32, on the native fp32 kernel."""
    x, y = _pair(x, y, "polynomial_kernel")
    batch, (m, d), n = x.shape[:-2], x.shape[-2:], y.shape[-2]
    if m == 0 or n == 0 or batch.numel() == 0:
        return x.new_empty(*batch, m, n)
    out = _native.polynomial_kernel(x.reshape(-1, m, d), y.reshape(-1, n, d))
    return out.reshape(*batch, m, n)


def _mmd_from_matrices(kxx, kyy, kxy):
    """term_1 + term_2 - term_3 of the unbiased squared MMD from the three kernel matrices (torch ops)"""
    m, n = kxx.shape[-1], kyy.shape[-1]
    off_xx = kxx.sum([-1, -2]) - kxx.diagonal(dim1=-2, dim2=-1).sum(-1)
    off_yy = kyy.sum([-1, -2]) - kyy.diagonal(dim1=-2, dim2=-1).sum(-1)
    return off_xx / m / (m - 1) + off_yy / n / (n - 1) - kxy.sum([-1, -2]) * 2 / m / n


def squared_mmd(x, y, kernel=polynomial_kernel):
    """Unbiased squared MMD between x [..., m, d] and y [..., n, d] -> [...] fp32.  With the default kernel, one native call covers
    every batch entry (polynomial kernel, fp64 sums).  Any other `kernel(a, b)` callable is evaluated on (x, x), (y, y) and (x, y)
    and the MMD formed from its matrices with torch ops, as the reference does."""
    x, y = _pair(x, y, "squared_mmd")
    if kernel is not polynomial_kernel:
        return _mmd_from_matrices(kernel(x, x), kernel(y, y), kernel(x, y))
    batch, (m, d), n = x.shape[:-2], x.shape[-2:], y.shape[-2]
    B = batch.numel()
    if B == 0:
        return x.new_empty(batch)
    sums = _native.mmd_sums(x.reshape(-1, d), y.reshape(-1, d), [b * m for b in range(B + 1)], [b * n for b in range(B + 1)])
    return sums[:, 3].float().reshape(batch)


def _partition_bounds(size, n_partitions):
    """Row bounds of kid's partitions, the reference's expression: Python's round (half to even) of i * size / n_partitions"""
    return [round(i * size / n_partitions) for i in range(n_partitions + 1)]


def kid(x, y, max_size=5000):
    """Kernel Inception Distance of x [m, d] and y [n, d]: the mean squared MMD over ceil(max(m, n) / max_size) partitions, with the
    reference's partition bounds.  One native call for every partition; the mean is taken in fp64 -> 0-d fp32."""
    x, y = _pair(x, y, "kid", ndim=2)
    n_partitions = math.ceil(max(x.shape[0] / max_size, y.shape[0] / max_size))
    sums = _native.mmd_sums(x, y, _partition_bounds(x.shape[0], n_partitions), _partition_bounds(y.shape[0], n_partitions))
    return (sums[:, 3].sum() / n_partitions).float()


class _MatrixSquareRootEig(torch.autograd.Function):
    """Square root of symmetric matrices through eigh: A = V diag(w) V^T -> V diag(sqrt|w|) V^T.  Its derivative solves the Sylvester
    equation S dS + dS S = dA in the eigenbasis: dA = V ((V^T G V) / (s_i + s_j)) V^T with s = sqrt|w|."""

    @staticmethod
    def forward(ctx, a):
        w, v = torch.linalg.eigh(a)
        ctx.save_for_backward(w, v)
        return v @ w.abs().sqrt().diag_embed() @ v.mT

    @staticmethod
    def backward(ctx, grad):
        w, v = ctx.saved_tensors
        s = w.abs().sqrt()
        return v @ ((v.mT @ grad @ v) / (s.unsqueeze(-1) + s.unsqueeze(-2))) @ v.mT


def sqrtm_eig(a):
    """Square root of a (batch of) symmetric matrices by eigendecomposition, differentiable (torch.linalg.eigh on a's device)."""
    if a.ndim < 2:
        raise RuntimeError('tensor of matrices must have at least 2 dimensions')
    if a.shape[-2] != a.shape[-1]:
        raise RuntimeError('tensor must be batches of square matrices')
    return _MatrixSquareRootEig.apply(a)


def fid(x, y, eps=1e-8):
    """Frechet distance between Gaussians fitted to x [m, d] and y [n, d] -> 0-d fp32.  The means and covariances come from the native
    kernel (fp64 column sums, fp32 products, exactly symmetric covariances); the d x d products and eigh run in torch, fp32 with TF32
    matmul off."""
    x, y = _pair(x, y, "fid", ndim=2)
    x_mean, x_cov = _native.feature_mean_cov(x)
    y_mean, y_cov = _native.feature_mean_cov(y)
    with utils.tf32_mode(matmul=False):
        mean_term = (x_mean - y_mean).pow(2).sum()
        eye = torch.eye(x_cov.shape[0], device=x_cov.device, dtype=x_cov.dtype) * eps
        x_cov, y_cov = x_cov + eye, y_cov + eye
        x_sqrt = sqrtm_eig(x_cov)
        cov_term = torch.trace(x_cov + y_cov - 2 * sqrtm_eig(x_sqrt @ y_cov @ x_sqrt))
    return mean_term + cov_term
