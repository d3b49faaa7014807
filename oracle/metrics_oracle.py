"""float64 restatement of the reference's scoring functions (k_diffusion/evaluation.py:93-161), written from the formulas in numpy:

    k(a, b)        = (a . b / d + 1)^3
    squared MMD    = sum_{i != j} k(x_i, x_j) / (m (m - 1)) + sum_{i != j} k(y_i, y_j) / (n (n - 1)) - 2 sum_{i, j} k(x_i, y_j) / (m n)
    KID            = mean of the squared MMD over ceil(max(m, n) / max_size) partitions, partition i holding rows
                     round(i * size / P) .. round((i + 1) * size / P) (Python's round, half to even)
    sqrt(A)        = V diag(sqrt|w|) V^T for A = V diag(w) V^T
    FID            = |mu_x - mu_y|^2 + tr(C_x + C_y - 2 sqrt(sqrt(C_x) C_y sqrt(C_x))), C = cov + eps I (unbiased covariance)
"""
import math

import numpy as np


def polynomial_kernel(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    return (x @ np.swapaxes(y, -1, -2) / x.shape[-1] + 1.0) ** 3


def mmd_terms(x, y):
    """(sum of k(x, x) off the diagonal, the same for y, sum of k(x, y), squared MMD) over the last two axes"""
    kxx, kyy, kxy = polynomial_kernel(x, x), polynomial_kernel(y, y), polynomial_kernel(x, y)
    m, n = kxx.shape[-1], kyy.shape[-1]
    sxx = kxx.sum((-1, -2)) - np.trace(kxx, axis1=-2, axis2=-1)
    syy = kyy.sum((-1, -2)) - np.trace(kyy, axis1=-2, axis2=-1)
    sxy = kxy.sum((-1, -2))
    with np.errstate(divide="ignore", invalid="ignore"):
        mmd = sxx / (m * (m - 1.0)) + syy / (n * (n - 1.0)) - 2.0 * sxy / (m * float(n))
    return sxx, syy, sxy, mmd


def squared_mmd(x, y):
    return mmd_terms(x, y)[3]


def partition_bounds(size, n_partitions):
    return [round(i * size / n_partitions) for i in range(n_partitions + 1)]


def kid(x, y, max_size=5000):
    P = math.ceil(max(len(x) / max_size, len(y) / max_size))
    bx, by = partition_bounds(len(x), P), partition_bounds(len(y), P)
    return sum(squared_mmd(x[bx[i]:bx[i + 1]], y[by[i]:by[i + 1]]) for i in range(P)) / P


def kid_terms(x, y, max_size=5000):
    """[(sxx, syy, sxy, mmd)] per kid partition"""
    P = math.ceil(max(len(x) / max_size, len(y) / max_size))
    bx, by = partition_bounds(len(x), P), partition_bounds(len(y), P)
    return [mmd_terms(x[bx[i]:bx[i + 1]], y[by[i]:by[i + 1]]) for i in range(P)]


def sqrtm_eig(a):
    w, v = np.linalg.eigh(np.asarray(a, np.float64))
    return (v * np.sqrt(np.abs(w))[..., None, :]) @ np.swapaxes(v, -1, -2)


def mean_cov(x):
    x = np.asarray(x, np.float64)
    mu = x.mean(0)
    xc = x - mu
    return mu, xc.T @ xc / (len(x) - 1)


def fid(x, y, eps=1e-8):
    mx, cx = mean_cov(x)
    my, cy = mean_cov(y)
    eye = np.eye(len(cx)) * eps
    cx, cy = cx + eye, cy + eye
    sx = sqrtm_eig(cx)
    return float(((mx - my) ** 2).sum() + np.trace(cx + cy - 2.0 * sqrtm_eig(sx @ cy @ sx)))
