"""Sigma schedules, noise samplers and the Karras ODE/SDE solver loops on H100-native kernels.

Drop-in for the functions of reference `k_diffusion/sampling.py` that are on the north-star path:
schedules (:17-43), `to_d` (:46), `get_ancestral_step` (:51), noise samplers (:61-114),
`sample_euler` (:117), `sample_euler_ancestral` (:138), `sample_heun` (:158), `sample_dpmpp_2m` (:584), and of the callers around it:
the other fixed-schedule samplers (:186-278, :519-700), DPM-Solver fast / adaptive (:303-516), the CFG wrapper of train.py:333-344.

How this differs from the reference implementation:
  * the sigma schedule is pulled to the host ONCE; every per-step coefficient is a host scalar, so
    the loop issues no device->host synchronisation (the reference syncs 2-3 times per step);
  * each solver stage is ONE fused 128-bit-vectorised kernel over the latent (libkdb200 solver ops)
    instead of 6-12 elementwise ATen kernels;
  * when `model` is `Denoiser(ImageTransformerDenoiserModelV2)` the conditioning of every model
    evaluation (mapping network + all AdaRMSNorm scales) is computed before the loop and the whole
    loop is replayed as one CUDA graph;
  * `sample_euler` / `sample_heun` only draw churn noise when gamma > 0 (the reference draws and
    discards `randn_like(x)` every step; samples are identical, the global RNG offset afterwards is not).
"""
import functools
import math
import os

import numpy as np
import torch

try:
    from tqdm.auto import trange
except ImportError:                                      # tqdm is optional plumbing
    def trange(n, disable=None):
        return range(n)

from . import _native, utils

f32 = np.float32


# --------------------------------------------------------------------------------------------
# schedules: same torch op sequence on the same device as the reference => bit-identical
# --------------------------------------------------------------------------------------------

def append_zero(x):
    return torch.cat([x, x.new_zeros([1])])


def get_sigmas_karras(n, sigma_min, sigma_max, rho=7., device='cpu'):
    """Karras et al. (2022) rho-schedule; ramp evaluated on the CPU, then moved (as the reference does)."""
    ramp = torch.linspace(0, 1, n)
    min_inv_rho = sigma_min ** (1 / rho)
    max_inv_rho = sigma_max ** (1 / rho)
    sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
    return append_zero(sigmas).to(device)


def get_sigmas_exponential(n, sigma_min, sigma_max, device='cpu'):
    """Log-linear schedule."""
    return append_zero(torch.linspace(math.log(sigma_max), math.log(sigma_min), n, device=device).exp())


def get_sigmas_polyexponential(n, sigma_min, sigma_max, rho=1., device='cpu'):
    """Polynomial-in-log-sigma schedule."""
    ramp = torch.linspace(1, 0, n, device=device) ** rho
    return append_zero(torch.exp(ramp * (math.log(sigma_max) - math.log(sigma_min)) + math.log(sigma_min)))


def get_sigmas_vp(n, beta_d=19.9, beta_min=0.1, eps_s=1e-3, device='cpu'):
    """Continuous VP schedule."""
    t = torch.linspace(1, eps_s, n, device=device)
    return append_zero(torch.sqrt(torch.exp(beta_d * t ** 2 / 2 + beta_min * t) - 1))


# --------------------------------------------------------------------------------------------
# solver primitives
# --------------------------------------------------------------------------------------------

def to_d(x, sigma, denoised):
    """Karras ODE derivative (x - denoised) / sigma; sigma 0-dim or [B]."""
    _native.require_cuda(x, denoised)
    sig = torch.as_tensor(sigma, dtype=torch.float32, device=x.device).reshape(-1)
    sig = sig.expand(x.shape[0]).contiguous()
    return _native.to_d(_native.f32c(x), _native.f32c(denoised), sig)


def get_ancestral_step(sigma_from, sigma_to, eta=1.):
    """(sigma_down, sigma_up) of an ancestral step; accepts tensors or floats."""
    if not eta:
        return sigma_to, 0.
    sigma_up = min(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


def default_noise_sampler(x):
    """Unit normal noise from torch's global generator (keeps `torch.manual_seed` reproducibility)."""
    return lambda sigma, sigma_next: torch.randn_like(x)


def _as_seed_tensor(seed, device):
    return torch.as_tensor(seed, dtype=torch.int64).reshape(-1).to(device)


class PhiloxNoiseSampler:
    """Counter-based unit normal noise: sample b, call k, element i -> Philox(seed[b]; k, i).

    Per-sample seeds make the noise independent of how a batch is sharded over GPUs."""

    def __init__(self, x, seeds, stream_base=1):
        self.like = x
        self.seeds = _as_seed_tensor(seeds, x.device)
        if self.seeds.numel() != x.shape[0]:
            raise ValueError("PhiloxNoiseSampler needs one seed per batch item")
        self.calls = 0
        self.stream_base = stream_base

    def __call__(self, sigma, sigma_next):
        self.calls += 1
        return _native.noise_normal(self.like, self.seeds, self.stream_base + self.calls)


class BatchedBrownianTree:
    """Brownian motion W on [t0, t1] per batch item, evaluated from counters instead of a host-side
    tree of cached nodes (reference wraps torchsde.BrownianTree, sampling.py:65-89).

    `tree(ta, tb)` returns W(tb) - W(ta) (sign handling as in the reference).  A list of seeds of
    length B gives every batch item its own path; a single seed drives one path over the whole tensor.
    Not bit-compatible with torchsde (absent here; parity unpinned) -- same law, different stream.
    """

    def __init__(self, x, t0, t1, seed=None, depth=24, **kwargs):
        _native.require_cuda(x)
        t0, t1 = float(t0), float(t1)
        self.t0, self.t1, self.sign = (t0, t1, 1) if t0 < t1 else (t1, t0, -1)
        if seed is None:
            seed = torch.randint(0, 2 ** 63 - 1, []).item()
        try:
            assert len(seed) == x.shape[0]
            self.batched = True
        except TypeError:
            seed = [seed]
            self.batched = False
        self.seeds = _as_seed_tensor(seed, x.device)
        self.like = x if self.batched else x.reshape(1, -1)
        self.shape = x.shape
        self.depth = depth
        if 'w0' in kwargs and kwargs['w0'] is not None and bool((kwargs['w0'] != 0).any()):
            raise ValueError("non-zero w0 is not supported")

    def normalized(self, ta, tb):
        """(W(tb) - W(ta)) / sqrt(|tb - ta|): unit-variance increments, one kernel."""
        ta, tb = float(ta), float(tb)
        if self.sign < 0:
            ta, tb = tb, ta
        return _native.noise_brownian(self.like, self.seeds, self.t0, self.t1, ta, tb, self.depth).view(self.shape)

    def __call__(self, t0, t1):
        w = self.normalized(t0, t1)
        return _native.lincomb([w], [math.sqrt(abs(float(t1) - float(t0)))])


class BrownianTreeNoiseSampler:
    """Noise sampler correlated across calls through one Brownian path per batch item
    (same constructor as reference sampling.py:92-114)."""

    def __init__(self, x, sigma_min, sigma_max, seed=None, transform=lambda x: x):
        self.transform = transform
        t0, t1 = self.transform(torch.as_tensor(sigma_min)), self.transform(torch.as_tensor(sigma_max))
        self.tree = BatchedBrownianTree(x, t0, t1, seed)

    def __call__(self, sigma, sigma_next):
        t0, t1 = self.transform(torch.as_tensor(sigma)), self.transform(torch.as_tensor(sigma_next))
        return self.tree.normalized(float(t0), float(t1))


# --------------------------------------------------------------------------------------------
# host-side step plans (pure Python/numpy: testable without a GPU)
# --------------------------------------------------------------------------------------------

def host_sigmas(sigmas):
    """The schedule as Python floats holding the exact fp32 values (one device->host copy)."""
    if sigmas.ndim != 1 or len(sigmas) < 2:
        raise ValueError("sigmas must be a 1-D tensor with at least two entries")
    return [float(v) for v in sigmas.detach().to(torch.float32).cpu().tolist()]


# Every fixed-schedule sampler is a plan: a list of steps, each a short list of ops over named buffers ('x' is the state):
#     ('eval',  out, src)                 out = D(src, sigma_k)      k-th entry of the step's 'evals'
#     ('lin',   out, [(name, coef), ...]) out = sum coef * name      one kdb_solver_lincomb launch
#     ('noise', out, sigma_from, sigma_to) out = noise_sampler(sigma_from, sigma_to)
#     ('randn', out)                      out = torch.randn_like(x)  torch's global generator (Karras churn): never captured
#     ('keep',  out, src)                 out aliases src (history of multistep methods; evals always write fresh buffers)
#     ('euler', out, x, den, r, noise, cn)          out = x + (x - den) r [+ noise cn]       one kdb_solver_euler_step launch
#     ('heun',  out, x, den, x2, den2, a1, a2)      out = x + (x - den) a1 + (x2 - den2) a2  one kdb_solver_heun_correct launch
#     ('dpmpp_2m', out, x, den, old, a, b, k1, k0)  out = a x - b (k1 den + k0 old)          one kdb_solver_dpmpp_2m_step launch
# In 'euler' noise = None drops the noise term; in 'dpmpp_2m' old is not read when k0 == 0 (the first step has no history).
# The fused kinds serve Euler, Heun, Euler-ancestral and DPM++(2M).  Every update of the other samplers is a linear combination,
# with host-computable scalar coefficients, of at most five image tensors: they stay on 'lin' (a fused kind would change their rounding).
# Plans are pure host math (verified on the CPU against reference trajectories in tests/test_host_logic.py); `_sample_ops` runs them.

def _churn(sig, i, s_churn, s_tmin, s_tmax, s_noise):
    """(gamma, sigma_hat, ops) of step i's Karras churn: the noise is drawn only on steps with gamma > 0 (DESIGN.md quirk Q1)."""
    n = len(sig) - 1
    gamma = min(s_churn / n, 2 ** 0.5 - 1) if s_tmin <= sig[i] <= s_tmax else 0.
    sigma_hat = float(f32(sig[i]) * f32(gamma + 1))
    if not gamma > 0:
        return gamma, sigma_hat, []
    coef = float(np.sqrt(f32(sigma_hat) ** 2 - f32(sig[i]) ** 2))
    return gamma, sigma_hat, [('randn', 'n'), ('lin', 'x', [('x', 1.), ('n', s_noise * coef)])]


def plan_euler(sig, s_churn=0., s_tmin=0., s_tmax=float('inf'), s_noise=1.):
    steps = []
    for i in range(len(sig) - 1):
        gamma, sigma_hat, ops = _churn(sig, i, s_churn, s_tmin, s_tmax, s_noise)
        r = float(f32(sig[i + 1]) - f32(sigma_hat)) / sigma_hat
        ops += [('eval', 'den', 'x'), ('euler', 'x', 'x', 'den', r, None, 0.)]
        steps.append(dict(i=i, gamma=gamma, sigma_hat=sigma_hat, ops=ops, evals=[sigma_hat]))
    return steps


def plan_heun(sig, s_churn=0., s_tmin=0., s_tmax=float('inf'), s_noise=1.):
    steps = []
    for i in range(len(sig) - 1):
        gamma, sigma_hat, ops = _churn(sig, i, s_churn, s_tmin, s_tmax, s_noise)
        nxt = sig[i + 1]
        dt = float(f32(nxt) - f32(sigma_hat))
        if nxt == 0:                                      # the final step to sigma = 0 is Euler
            ops += [('eval', 'den', 'x'), ('euler', 'x', 'x', 'den', dt / sigma_hat, None, 0.)]
            evals = [sigma_hat]
        else:                                             # Euler predictor, trapezoidal corrector
            ops += [('eval', 'den', 'x'), ('euler', 'x2', 'x', 'den', dt / sigma_hat, None, 0.), ('eval', 'den2', 'x2'),
                    ('heun', 'x', 'x', 'den', 'x2', 'den2', dt / (2 * sigma_hat), dt / (2 * nxt))]
            evals = [sigma_hat, nxt]
        steps.append(dict(i=i, gamma=gamma, sigma_hat=sigma_hat, ops=ops, evals=evals))
    return steps


def plan_euler_ancestral(sig, eta=1., s_noise=1.):
    steps = []
    for i in range(len(sig) - 1):
        down, up = get_ancestral_step(sig[i], sig[i + 1], eta=eta)
        noise = [('noise', 'n', sig[i], sig[i + 1])] if sig[i + 1] > 0 else []
        ops = [('eval', 'den', 'x')] + noise + [('euler', 'x', 'x', 'den', (down - sig[i]) / sig[i], 'n' if noise else None, s_noise * up)]
        steps.append(dict(i=i, sigma_hat=sig[i], ops=ops, evals=[sig[i]]))
    return steps


def plan_dpmpp_2m(sig):
    steps = []
    for i in range(len(sig) - 1):
        s, s_next = sig[i], sig[i + 1]
        if s_next == 0:
            a, b, h = 0., -1., math.inf                       # expm1(-inf) = -1, sigma_next/sigma = 0
        else:
            h = math.log(s) - math.log(s_next)
            a, b = s_next / s, math.expm1(-h)
        if i == 0 or s_next == 0:
            k1, k0 = 1., 0.
        else:
            r = (math.log(sig[i - 1]) - math.log(s)) / h
            k1, k0 = 1 + 1 / (2 * r), -1 / (2 * r)
        ops = [('eval', 'den', 'x'), ('dpmpp_2m', 'x', 'x', 'den', 'old', a, b, k1, k0), ('keep', 'old', 'den')]
        steps.append(dict(i=i, sigma_hat=s, ops=ops, evals=[s]))
    return steps


def _log_mid(a, b):
    return math.exp(0.5 * (math.log(a) + math.log(b)))


def _euler_to(target, sigma):
    """x + (x - den) / sigma * (target - sigma) as coefficients on (x, den)."""
    r = (target - sigma) / sigma
    return [('x', 1 + r), ('den', -r)]


def _dpm2_ops(sigma, target):
    """DPM-Solver-2 step from sigma to target (midpoint in log sigma), sampling.py:205-214 / :233-242."""
    if target == 0:
        return [('eval', 'den', 'x'), ('lin', 'x', _euler_to(target, sigma))], [sigma]
    mid = _log_mid(sigma, target)
    r1, c2 = (mid - sigma) / sigma, (target - sigma) / mid
    return [('eval', 'den', 'x'), ('lin', 'x2', [('x', 1 + r1), ('den', -r1)]), ('eval', 'den2', 'x2'),
            ('lin', 'x', [('x', 1.), ('x2', c2), ('den2', -c2)])], [sigma, mid]


def plan_dpm_2(sig, s_churn=0., s_tmin=0., s_tmax=float('inf'), s_noise=1.):
    steps = []
    for i in range(len(sig) - 1):
        gamma, sigma_hat, churn = _churn(sig, i, s_churn, s_tmin, s_tmax, s_noise)
        ops, evals = _dpm2_ops(sigma_hat, sig[i + 1])
        steps.append(dict(i=i, gamma=gamma, sigma_hat=sigma_hat, ops=churn + ops, evals=evals))
    return steps


def plan_dpm_2_ancestral(sig, eta=1., s_noise=1.):
    steps = []
    for i in range(len(sig) - 1):
        down, up = get_ancestral_step(sig[i], sig[i + 1], eta=eta)
        ops, evals = _dpm2_ops(sig[i], down)
        if down != 0:
            ops += [('noise', 'n', sig[i], sig[i + 1]), ('lin', 'x', [('x', 1.), ('n', s_noise * up)])]
        steps.append(dict(i=i, sigma_hat=sig[i], ops=ops, evals=evals))
    return steps


def lms_coefficient(order, t, i, j):
    """Integral over [t_i, t_{i+1}] of the j-th Lagrange basis polynomial through t_i, t_{i-1}, ... (sampling.py:247-257).
    Degree order - 1, so Gauss-Legendre with >= order / 2 nodes is exact (the reference uses scipy quad with epsrel 1e-4)."""
    if order - 1 > i:
        raise ValueError(f'Order {order} too high for step {i}')
    a, b = t[i], t[i + 1]
    nodes, weights = np.polynomial.legendre.leggauss(max(4, (order + 1) // 2))
    tau = 0.5 * (b - a) * nodes + 0.5 * (b + a)
    basis = np.ones_like(tau)
    for k in range(order):
        if k != j:
            basis = basis * (tau - t[i - k]) / (t[i - j] - t[i - k])
    return float(0.5 * (b - a) * np.dot(weights, basis))


linear_multistep_coeff = lms_coefficient        # the reference's name (sampling.py:247)


def plan_lms(sig, order=4):
    if order < 1:
        raise ValueError('order must be at least 1')
    steps = []
    for i in range(len(sig) - 1):
        cur = min(i + 1, order)
        # derivative ring d0 .. d{order-1}: rotate names instead of moving data (x + more than five derivatives: chained launches)
        names = [f'd{(i - j) % order}' for j in range(cur)]
        ops = [('eval', 'den', 'x'), ('lin', names[0], [('x', 1 / sig[i]), ('den', -1 / sig[i])]),
               ('lin', 'x', [('x', 1.)] + [(names[j], lms_coefficient(cur, sig, i, j)) for j in range(cur)])]
        steps.append(dict(i=i, sigma_hat=sig[i], ops=ops, evals=[sig[i]]))
    return steps


def plan_dpmpp_2s_ancestral(sig, eta=1., s_noise=1.):
    steps = []
    for i in range(len(sig) - 1):
        s = sig[i]
        down, up = get_ancestral_step(s, sig[i + 1], eta=eta)
        if down == 0:
            ops, evals = [('eval', 'den', 'x'), ('lin', 'x', _euler_to(down, s))], [s]
        else:
            h = math.log(s) - math.log(down)                       # t_next - t with t = -log sigma
            mid = math.exp(-(-math.log(s) + 0.5 * h))
            ops = [('eval', 'den', 'x'), ('lin', 'x2', [('x', mid / s), ('den', -math.expm1(-0.5 * h))]), ('eval', 'den2', 'x2'),
                   ('lin', 'x', [('x', down / s), ('den2', -math.expm1(-h))])]
            evals = [s, mid]
        if sig[i + 1] > 0:
            ops += [('noise', 'n', s, sig[i + 1]), ('lin', 'x', [('x', 1.), ('n', s_noise * up)])]
        steps.append(dict(i=i, sigma_hat=s, ops=ops, evals=evals))
    return steps


def _exp_step(sigma, down):
    """(ratio, expm1(t - t_down)) of the exponential-integrator update towards sigma = down, with the down == 0 limit."""
    if down == 0:
        return 0., -1.
    return down / sigma, math.expm1(math.log(down) - math.log(sigma))


def plan_dpmpp_sde(sig, eta=1., s_noise=1., r=1 / 2):
    steps = []
    for i in range(len(sig) - 1):
        s, s_next = sig[i], sig[i + 1]
        if s_next == 0:
            steps.append(dict(i=i, sigma_hat=s, ops=[('eval', 'den', 'x'), ('lin', 'x', _euler_to(0., s))], evals=[s]))
            continue
        t, t_next = -math.log(s), -math.log(s_next)
        h = t_next - t
        mid = math.exp(-(t + h * r))
        fac = 1 / (2 * r)
        sd, su = get_ancestral_step(s, mid, eta)
        ratio1, e1 = _exp_step(s, sd)
        sd2, su2 = get_ancestral_step(s, s_next, eta)
        ratio2, e2 = _exp_step(s, sd2)
        ops = [('eval', 'den', 'x'), ('noise', 'n', s, mid),
               ('lin', 'x2', [('x', ratio1), ('den', -e1), ('n', s_noise * su)]), ('eval', 'den2', 'x2'), ('noise', 'n', s, s_next),
               ('lin', 'x', [('x', ratio2), ('den', -e2 * (1 - fac)), ('den2', -e2 * fac), ('n', s_noise * su2)])]
        steps.append(dict(i=i, sigma_hat=s, ops=ops, evals=[s, mid]))
    return steps


def plan_dpmpp_2m_sde(sig, eta=1., s_noise=1., solver_type='midpoint'):
    if solver_type not in {'heun', 'midpoint'}:
        raise ValueError('solver_type must be \'heun\' or \'midpoint\'')
    steps, h_last = [], None
    for i in range(len(sig) - 1):
        s, s_next = sig[i], sig[i + 1]
        if s_next == 0:
            ops = [('eval', 'den', 'x'), ('lin', 'x', [('den', 1.)])]
        else:
            h = math.log(s) - math.log(s_next)
            eta_h = eta * h
            gain = -math.expm1(-h - eta_h)
            terms = {'x': s_next / s * math.exp(-eta_h), 'den': gain}
            if h_last is not None:
                r = h_last / h
                corr = (gain / (-h - eta_h) + 1) / r if solver_type == 'heun' else 0.5 * gain / r
                terms['den'] += corr
                terms['old'] = -corr
            ops = [('eval', 'den', 'x')]
            if eta:
                ops.append(('noise', 'n', s, s_next))
                terms['n'] = s_next * math.sqrt(-math.expm1(-2 * eta_h)) * s_noise
            ops.append(('lin', 'x', list(terms.items())))
            h_last = h
        ops.append(('keep', 'old', 'den'))
        steps.append(dict(i=i, sigma_hat=s, ops=ops, evals=[s]))
    return steps


def plan_dpmpp_3m_sde(sig, eta=1., s_noise=1.):
    steps, h_1, h_2 = [], None, None
    for i in range(len(sig) - 1):
        s, s_next = sig[i], sig[i + 1]
        h = None
        if s_next == 0:
            ops = [('eval', 'den', 'x'), ('lin', 'x', [('den', 1.)])]
        else:
            h = math.log(s) - math.log(s_next)
            h_eta = h * (eta + 1)
            terms = {'x': math.exp(-h_eta), 'den': -math.expm1(-h_eta)}
            if h_2 is not None:
                r0, r1 = h_1 / h, h_2 / h
                phi_2 = math.expm1(-h_eta) / h_eta + 1
                phi_3 = phi_2 / h_eta - 0.5
                q, w = r0 / (r0 + r1), 1 / (r0 + r1)
                ca, cb = phi_2 * (1 + q) - phi_3 * w, phi_2 * q - phi_3 * w      # coefficients of d1_0 and (minus) d1_1
                terms['den'] += ca / r0
                terms['old'] = -ca / r0 - cb / r1
                terms['old2'] = cb / r1
            elif h_1 is not None:
                phi_2 = math.expm1(-h_eta) / h_eta + 1
                terms['den'] += phi_2 / (h_1 / h)
                terms['old'] = -phi_2 / (h_1 / h)
            ops = [('eval', 'den', 'x')]
            if eta:
                ops.append(('noise', 'n', s, s_next))
                terms['n'] = s_next * math.sqrt(-math.expm1(-2 * h * eta)) * s_noise
            ops.append(('lin', 'x', list(terms.items())))
        ops += ([('keep', 'old2', 'old')] if i > 0 else []) + [('keep', 'old', 'den')]     # aliases, no copies
        h_1, h_2 = h, h_1
        steps.append(dict(i=i, sigma_hat=s, ops=ops, evals=[s]))
    return steps


# --------------------------------------------------------------------------------------------
# classifier-free guidance (SURVEY 8f.2; reference train.py:333-344 make_cfg_model_fn)
# --------------------------------------------------------------------------------------------

class CFGDenoiser:
    """model_fn(x, sigma, class_cond) = uncond + (cond - uncond) * cfg_scale on a doubled batch [uncond | cond].

    `num_classes` is the index of the unconditional token (class_emb has num_classes + 1 rows, reference config.py:208).
    Called directly it works around ANY `model(x, sigma, class_cond=...)`.  Passed to a sampler of this package with a native
    `Denoiser` inside, the sampler evaluates the doubled batch in one engine call per step (conditioning rows of all steps
    precomputed) and the whole loop, guidance included, is captured into one CUDA graph."""

    def __init__(self, model, cfg_scale, num_classes):
        self.inner_model, self.cfg_scale, self.num_classes = model, float(cfg_scale), int(num_classes)

    def double(self, x, sigma, class_cond):
        return torch.cat([x, x]), torch.cat([sigma, sigma]), torch.cat([torch.full_like(class_cond, self.num_classes), class_cond])

    def __call__(self, x, sigma, class_cond):
        x_in, sigma_in, cc = self.double(x, sigma, class_cond)
        out = self.inner_model(x_in, sigma_in, class_cond=cc)
        out_uncond, out_cond = out.chunk(2)
        if not out.is_cuda:
            raise RuntimeError("k_diffusion (H100-native) operates on CUDA tensors only; there is no CPU fallback")
        return _native.cfg_combine(_native.f32c(out_uncond), _native.f32c(out_cond), self.cfg_scale)


def make_cfg_model_fn(model, cfg_scale, num_classes):
    """Same contract as the closure in reference train.py:333-344: returns `model` itself when cfg_scale == 1."""
    return CFGDenoiser(model, cfg_scale, num_classes) if cfg_scale != 1 else model


# --------------------------------------------------------------------------------------------
# loop runner
# --------------------------------------------------------------------------------------------

_NATIVE_KW = {"aug_cond", "class_cond", "mapping_cond"}
_GRAPH_ENV = "KDB200_CUDA_GRAPH"


_COND_TABLE_BYTES = 1 << 30         # precompute the per-sample conditioning rows of ALL evaluations up to this size


class _Evaluator:
    """denoised = D(x, sigma_k) for the k-th model evaluation of a plan."""

    def __init__(self, model, x, extra_args, eval_sigmas):
        from .layers import Denoiser
        self.cfg = model if isinstance(model, CFGDenoiser) else None
        base = model.inner_model if self.cfg is not None else model
        self.model, self.extra_args = model, extra_args
        self.B = x.shape[0]
        keys_ok = set(extra_args) == {"class_cond"} if self.cfg is not None else set(extra_args) <= _NATIVE_KW
        self.native = isinstance(base, Denoiser) and base.is_native() and keys_ok
        sig = torch.tensor(eval_sigmas, dtype=torch.float32, device=x.device)
        self.sigma_rows = sig[:, None].expand(len(eval_sigmas), self.B).contiguous()
        if self.native:
            self.inner = base.inner_model
            self.call = self.inner.native_eval(x, None, **extra_args)      # every check of the inputs, once per sampler call
            if self.cfg is not None:
                self.call.guide(self.cfg.num_classes)
            self.eng, self.precision = self.call.engine, self.call.precision
            self.sigma_data = float(base.sigma_data)
            self.per_sample = any(extra_args.get(k) is not None for k in _NATIVE_KW)
            self._sig_rows, self.table = sig, None                               # conditioning table: built on first use
            self.n_evals = len(eval_sigmas)
            if self.cfg is not None:                                             # doubled batch: [uncond | cond]
                self.sigma_rows2 = sig[:, None].expand(self.n_evals, 2 * self.B).contiguous()
                self._x2 = None

    def capturable(self):
        return self.native

    def graph_tag(self):
        return ("cfg", self.cfg.cfg_scale, self.cfg.num_classes) if self.native and self.cfg is not None else ()

    def static_args(self):
        """The per-sample conditioning tensors a captured graph reads ((name, tensor) pairs, stable order)."""
        return [(k, self.extra_args[k]) for k in sorted(_NATIVE_KW) if self.native and self.extra_args.get(k) is not None]

    def _cond_args(self, reps):
        """aug / class / mapping conditioning tensors for `reps` evaluations (the doubled CFG batch included), read from extra_args, which
        a graph capture points at its static copies."""
        ea = self.extra_args
        return self.call.cond_args(reps, ea.get("aug_cond"), ea.get("class_cond"), ea.get("mapping_cond"))

    def _per_sample_rows(self, k, rows):
        """Conditioning rows [rows, stride] of evaluation k.  All evaluations' rows come from ONE launch when they fit the
        table budget (the conditioning kernel is a latency-bound chain of mat-vecs: ~1.5 ms whether it serves 64 rows or 6000)."""
        stride = self.eng.cond_stride
        sig_rows = self.sigma_rows2 if self.cfg is not None else self.sigma_rows
        if self.n_evals * rows * stride * 4 <= _COND_TABLE_BYTES:
            if self.table is None:
                aug, cc, mc = self._cond_args(self.n_evals)
                self.table = self.eng.conditioning(sig_rows.reshape(-1), aug, cc, mc)
            return self.table[k * rows:(k + 1) * rows]
        aug, cc, mc = self._cond_args(1)
        return self.eng.conditioning(sig_rows[k], aug, cc, mc)

    def __call__(self, k, x, out=None):
        if not self.native:
            return self.model(x, self.sigma_rows[k], **self.extra_args)
        if self.cfg is not None:
            if self._x2 is None or self._x2.shape[0] != 2 * self.B:
                self._x2 = torch.empty(2 * self.B, *x.shape[1:], device=x.device, dtype=torch.float32)
            torch.cat([x, x], out=self._x2)
            cond = self._per_sample_rows(k, 2 * self.B)
            both = self.eng.forward(self._x2, self.sigma_rows2[k], cond, self.eng.cond_stride, self.sigma_data, self.precision)
            return _native.cfg_combine(both[:self.B], both[self.B:], self.cfg.cfg_scale, out=out)
        cond, stride = self._rows(k)
        return self.eng.forward(x, self.sigma_rows[k], cond, stride, self.sigma_data, self.precision, out=out)

    def _rows(self, k):
        """(conditioning rows, batch stride) of evaluation k without CFG"""
        if self.per_sample:
            return self._per_sample_rows(k, self.B), self.eng.cond_stride
        if self.table is None:              # one launch for every evaluation of the schedule (a cached graph never needs it)
            self.table = self.eng.conditioning(self._sig_rows)
        return self.table[k], 0

    def jvp(self, k, x, v):
        """(D(x, sigma_k), J_D(x) v): one forward-mode engine call on the fp32 path (native, without CFG)"""
        cond, stride = self._rows(k)
        return self.eng.forward_jvp(x, v, self.sigma_rows[k], cond, stride, self.sigma_data)

    def vjp(self, k, x, u):
        """(D(x, sigma_k), u^T J_D(x)): one reverse-mode engine call on the fp32 path (native, without CFG)"""
        cond, stride = self._rows(k)
        return self.eng.forward_vjp(x, u, self.sigma_rows[k], cond, stride, self.sigma_data)


def _prepare(x, sigmas, extra_args):
    _native.require_cuda(x)
    extra_args = {} if extra_args is None else extra_args
    return _native.f32c(x), host_sigmas(sigmas), extra_args


def _finish(x_work, x):
    return x_work if x.dtype == torch.float32 else x_work.to(x.dtype)


def _scalar_like(sigmas, v):
    """0-d tensor of v on sigmas' device, filled there: a host-to-device copy would synchronise the eager loop every step"""
    return torch.full((), v, dtype=sigmas.dtype, device=sigmas.device)


_graph_cache = {}
_GLOBAL_RNG = object()          # marker: the body draws from torch's global generator -> never captured


def _progress(plan, disable):
    """tqdm over the steps in eager mode; plain iteration while a CUDA graph is being captured/warmed."""
    if disable or torch.cuda.is_current_stream_capturing() or _progress.quiet:
        return plan
    idx = trange(len(plan), disable=disable)
    return (plan[i] for i in idx)


_progress.quiet = False


def _noise_kind(noise_sampler):
    """How a noise sampler may be used inside a captured graph.

    'none'      no noise is drawn
    'brownian'  BrownianTreeNoiseSampler: a pure function of (seeds, sigma, sigma_next) -> capturable; the seeds live in a
                static device buffer owned by the cache entry and are refreshed before every replay, so one graph serves
                every seed (and a sampler that was freed can never be replayed by address)
    'foreign'   anything else (global-RNG randn, PhiloxNoiseSampler's call counter, user callables): eager only
    """
    if noise_sampler is None:
        return 'none'
    if isinstance(noise_sampler, BrownianTreeNoiseSampler):
        return 'brownian'
    return 'foreign'


def _graph_key(name, ev, x, sig, params, noise_sampler):
    key = (name, id(ev.inner), ev.eng._sig, ev.sigma_data, tuple(x.shape), x.device.index, tuple(sig), ev.precision, params,
           tuple((k, tuple(t.shape), str(t.dtype)) for k, t in ev.static_args()), ev.graph_tag())
    if _noise_kind(noise_sampler) == 'brownian':
        tr = noise_sampler.tree          # the entry keeps `transform` alive, so its id cannot be recycled while the key exists
        key += (('brownian', tr.t0, tr.t1, tr.sign, tr.depth, tr.batched, int(tr.seeds.numel()), id(noise_sampler.transform)),)
    return key


class _GraphEntry:
    """One captured sampler call.  Holds every object whose ADDRESS the graph (or its key) depends on."""
    __slots__ = ("graph", "static_in", "static_out", "kernels", "ev", "ws", "static_args", "static_seeds", "transform")


def _run(name, body, ev, x, sig, params, callback, noise_sampler=None):
    """Run `body(x) -> x_out` eagerly, or as a cached CUDA graph when everything inside is ours."""
    kind = _noise_kind(noise_sampler)
    use_graph = (os.environ.get(_GRAPH_ENV, "1") != "0" and callback is None and ev.capturable() and kind != 'foreign'
                 and not torch.cuda.is_current_stream_capturing())
    if not use_graph:
        return body(x)
    key = _graph_key(name, ev, x, sig, params, noise_sampler)
    entry = _graph_cache.get(key)
    if entry is None:
        entry = _GraphEntry()
        entry.static_in = torch.empty_like(x)
        entry.static_in.copy_(x)
        # per-sample conditioning tensors and Brownian seeds are read through static copies owned by the entry
        entry.static_args = {k: t.clone() for k, t in ev.static_args()}
        entry.static_seeds = noise_sampler.tree.seeds.clone() if kind == 'brownian' else None
        entry.transform = noise_sampler.transform if kind == 'brownian' else None
        call_args, ev.extra_args = ev.extra_args, {**ev.extra_args, **entry.static_args}
        if kind == 'brownian':
            call_seeds, noise_sampler.tree.seeds = noise_sampler.tree.seeds, entry.static_seeds
        side = torch.cuda.Stream(device=x.device)
        side.wait_stream(torch.cuda.current_stream())
        _progress.quiet = True
        try:
            with torch.cuda.stream(side):                  # warm-up outside capture (allocations, pos tables)
                body(entry.static_in)
            torch.cuda.current_stream().wait_stream(side)
            if ev.static_args():
                ev.table = None      # per-sample conditioning rows depend on the (refreshable) labels: their launch belongs INSIDE the graph
            entry.graph = torch.cuda.CUDAGraph()
            n0 = _native.launch_count()
            with torch.cuda.graph(entry.graph):
                entry.static_out = body(entry.static_in)
            entry.kernels = _native.launch_count() - n0        # kernel nodes of ours inside the graph
        finally:
            _progress.quiet = False
            ev.extra_args = call_args
            if kind == 'brownian':
                noise_sampler.tree.seeds = call_seeds
        entry.ev, entry.ws = ev, ev.eng._ws                    # keeps the model, its engine and the workspace alive
        if len(_graph_cache) >= int(os.environ.get("KDB200_GRAPH_CACHE", "8")):
            _graph_cache.pop(next(iter(_graph_cache)))
        _graph_cache[key] = entry
    entry.static_in.copy_(x)
    for k, t in ev.static_args():
        entry.static_args[k].copy_(t)
    if kind == 'brownian':
        entry.static_seeds.copy_(noise_sampler.tree.seeds)
    entry.graph.replay()
    _replayed[0] += entry.kernels
    return entry.static_out.clone()


_replayed = [0]


def total_kernel_launches():
    """Kernels of libkdb200 launched by this process: direct launches + kernel nodes of replayed graphs."""
    return _native.launch_count() + _replayed[0]


def clear_graph_cache():
    _graph_cache.clear()


# --------------------------------------------------------------------------------------------
# samplers
# --------------------------------------------------------------------------------------------

def _on_x_device(fn):
    """Run a sampler with x's GPU as the current device: kernels launch on the current device's current stream and the engine
    allocates its tables there, so `x` on cuda:1 under current device cuda:0 must switch (the reference's ATen ops do)."""
    @functools.wraps(fn)
    def wrapper(model, x, *args, **kwargs):
        with _native.device_of(x):
            return fn(model, x, *args, **kwargs)
    return wrapper


def _exec_op(op, T, ev, k, draw=None):
    """Execute one plan op on the named buffers T; `k` indexes the next model evaluation and `draw(sigma_from, sigma_to)` makes the
    noise of 'noise' ops.  Returns the number of model evaluations made (1 for 'eval', else 0)."""
    kind = op[0]
    if kind == 'eval':
        T[op[1]] = ev(k, T[op[2]])
        return 1
    if kind == 'lin':
        T[op[1]] = _lin_x([(T[n], c) for n, c in op[2]], keep_zero=True)
    elif kind == 'euler':
        T[op[1]] = _native.euler_step(T[op[2]], T[op[3]], op[4], noise=None if op[5] is None else T[op[5]], cn=op[6])
    elif kind == 'heun':
        T[op[1]] = _native.heun_correct(T[op[2]], T[op[3]], T[op[4]], T[op[5]], op[6], op[7])
    elif kind == 'dpmpp_2m':
        T[op[1]] = _native.dpmpp_2m_step(T[op[2]], T[op[3]], T[op[4]] if op[8] != 0 else None, *op[5:])
    elif kind == 'noise':
        T[op[1]] = _native.f32c(draw(op[2], op[3]))
    elif kind == 'randn':
        T[op[1]] = torch.randn_like(T['x'])
    else:                    # 'keep': alias, evaluations always write fresh buffers
        T[op[1]] = T[op[2]]
    return 0


def _sample_ops(name, model, x, sigmas, plan_fn, extra_args, callback, disable, params, noise_sampler=None, callback_extra=None, on_eval=None):
    """Run an op plan.  `plan_fn(sig)` builds it from the host copy of `sigmas` (or is the plan itself, a list);
    `callback_extra(st)` may add keys to the callback payload of a step; `on_eval()` runs after every model evaluation (like `callback`
    it keeps the loop out of a CUDA graph)."""
    xw, sig, extra_args = _prepare(x, sigmas, extra_args)
    plan = plan_fn if isinstance(plan_fn, list) else plan_fn(sig)
    kinds = {op[0] for st in plan for op in st['ops']}
    ours = isinstance(noise_sampler, (BrownianTreeNoiseSampler, PhiloxNoiseSampler))
    ev = _Evaluator(model, xw, extra_args, [s_ for st in plan for s_ in st['evals']])

    def draw(sigma_from, sigma_to):      # our samplers take host floats (no sync); foreign callables get tensors like the reference
        args = (sigma_from, sigma_to) if ours else (_scalar_like(sigmas, sigma_from), _scalar_like(sigmas, sigma_to))
        return noise_sampler(*args)

    def body(xc):
        T = {'x': xc}
        k = 0
        for st in _progress(plan, disable):
            first = True
            for op in st['ops']:
                k += _exec_op(op, T, ev, k, draw)
                if op[0] == 'eval':
                    if on_eval is not None:
                        on_eval()
                    if first and callback is not None:
                        callback({'x': T[op[2]], 'i': st['i'], 'sigma': sigmas[st['i']], 'sigma_hat': _scalar_like(sigmas, st['sigma_hat']),
                                  'denoised': T[op[1]], **({} if callback_extra is None else callback_extra(st))})
                    first = False
        return T['x']

    # a graph replays the same noise kernels every call: only legal without noise or with the Brownian tree
    out = _run(name, body, ev, xw, sig, params, callback if callback is not None else on_eval,
               noise_sampler=_GLOBAL_RNG if 'randn' in kinds else (noise_sampler if 'noise' in kinds else None))
    return _finish(out, x)


@_on_x_device
@torch.no_grad()
def sample_euler(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0., s_tmin=0., s_tmax=float('inf'), s_noise=1.):
    """Algorithm 2 (Euler steps) from Karras et al. (2022)."""
    return _sample_ops('euler', model, x, sigmas, lambda sig: plan_euler(sig, s_churn, s_tmin, s_tmax, s_noise), extra_args, callback, disable,
                       (s_churn, s_tmin, s_tmax, s_noise))


@_on_x_device
@torch.no_grad()
def sample_euler_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1., s_noise=1., noise_sampler=None):
    """Ancestral sampling with Euler method steps."""
    noise_sampler = default_noise_sampler(_native.f32c(x)) if noise_sampler is None else noise_sampler
    return _sample_ops('euler_a', model, x, sigmas, lambda sig: plan_euler_ancestral(sig, eta, s_noise), extra_args, callback, disable,
                       (eta, s_noise), noise_sampler)


@_on_x_device
@torch.no_grad()
def sample_heun(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0., s_tmin=0., s_tmax=float('inf'), s_noise=1.):
    """Algorithm 2 (Heun steps) from Karras et al. (2022)."""
    return _sample_ops('heun', model, x, sigmas, lambda sig: plan_heun(sig, s_churn, s_tmin, s_tmax, s_noise), extra_args, callback, disable,
                       (s_churn, s_tmin, s_tmax, s_noise))


@_on_x_device
@torch.no_grad()
def sample_dpmpp_2m(model, x, sigmas, extra_args=None, callback=None, disable=None):
    """DPM-Solver++(2M)."""
    return _sample_ops('dpmpp_2m', model, x, sigmas, plan_dpmpp_2m, extra_args, callback, disable, ())


def _default_brownian(x, sigmas):
    sigma_min, sigma_max = sigmas[sigmas > 0].min(), sigmas.max()
    return BrownianTreeNoiseSampler(_native.f32c(x), sigma_min, sigma_max)


@_on_x_device
@torch.no_grad()
def sample_dpm_2(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0., s_tmin=0., s_tmax=float('inf'), s_noise=1.):
    """A sampler inspired by DPM-Solver-2 and Algorithm 2 from Karras et al. (2022)  (reference sampling.py:187-214)."""
    return _sample_ops('dpm_2', model, x, sigmas, lambda sig: plan_dpm_2(sig, s_churn, s_tmin, s_tmax, s_noise), extra_args, callback, disable,
                       (s_churn, s_tmin, s_tmax, s_noise))


@_on_x_device
@torch.no_grad()
def sample_dpm_2_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1., s_noise=1., noise_sampler=None):
    """Ancestral sampling with DPM-Solver second-order steps  (reference sampling.py:217-244)."""
    noise_sampler = default_noise_sampler(_native.f32c(x)) if noise_sampler is None else noise_sampler
    return _sample_ops('dpm_2_a', model, x, sigmas, lambda sig: plan_dpm_2_ancestral(sig, eta, s_noise), extra_args, callback, disable,
                       (eta, s_noise), noise_sampler)


@_on_x_device
@torch.no_grad()
def sample_lms(model, x, sigmas, extra_args=None, callback=None, disable=None, order=4):
    """Linear multistep (Adams-Bashforth in sigma)  (reference sampling.py:247-277)."""
    return _sample_ops('lms', model, x, sigmas, lambda sig: plan_lms(sig, order), extra_args, callback, disable, (order,))


@_on_x_device
@torch.no_grad()
def sample_dpmpp_2s_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1., s_noise=1., noise_sampler=None):
    """Ancestral sampling with DPM-Solver++(2S) second-order steps  (reference sampling.py:508-539)."""
    noise_sampler = default_noise_sampler(_native.f32c(x)) if noise_sampler is None else noise_sampler
    return _sample_ops('dpmpp_2s_a', model, x, sigmas, lambda sig: plan_dpmpp_2s_ancestral(sig, eta, s_noise), extra_args, callback, disable,
                       (eta, s_noise), noise_sampler)


@_on_x_device
@torch.no_grad()
def sample_dpmpp_sde(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1., s_noise=1., noise_sampler=None, r=1 / 2):
    """DPM-Solver++ (stochastic)  (reference sampling.py:542-581)."""
    noise_sampler = _default_brownian(x, sigmas) if noise_sampler is None else noise_sampler
    return _sample_ops('dpmpp_sde', model, x, sigmas, lambda sig: plan_dpmpp_sde(sig, eta, s_noise, r), extra_args, callback, disable,
                       (eta, s_noise, r), noise_sampler)


@_on_x_device
@torch.no_grad()
def sample_dpmpp_2m_sde(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1., s_noise=1., noise_sampler=None,
                        solver_type='midpoint'):
    """DPM-Solver++(2M) SDE  (reference sampling.py:610-652)."""
    if solver_type not in {'heun', 'midpoint'}:
        raise ValueError('solver_type must be \'heun\' or \'midpoint\'')
    noise_sampler = _default_brownian(x, sigmas) if noise_sampler is None else noise_sampler
    return _sample_ops('dpmpp_2m_sde', model, x, sigmas, lambda sig: plan_dpmpp_2m_sde(sig, eta, s_noise, solver_type), extra_args, callback,
                       disable, (eta, s_noise, solver_type), noise_sampler)


@_on_x_device
@torch.no_grad()
def sample_dpmpp_3m_sde(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1., s_noise=1., noise_sampler=None):
    """DPM-Solver++(3M) SDE  (reference sampling.py:655-703)."""
    noise_sampler = _default_brownian(x, sigmas) if noise_sampler is None else noise_sampler
    return _sample_ops('dpmpp_3m_sde', model, x, sigmas, lambda sig: plan_dpmpp_3m_sde(sig, eta, s_noise), extra_args, callback, disable,
                       (eta, s_noise), noise_sampler)


# --------------------------------------------------------------------------------------------
# DPM-Solver: fixed-step "fast" and adaptive 12 / 23 (reference sampling.py:303-516)
# --------------------------------------------------------------------------------------------

class PIDStepSizeController:
    """A PID controller for ODE adaptive step size control (reference sampling.py:303-330; pure host arithmetic)."""

    def __init__(self, h, pcoeff, icoeff, dcoeff, order=1, accept_safety=0.81, eps=1e-8):
        self.h = h
        self.b1 = (pcoeff + icoeff + dcoeff) / order
        self.b2 = -(pcoeff + 2 * dcoeff) / order
        self.b3 = dcoeff / order
        self.accept_safety = accept_safety
        self.eps = eps
        self.errs = []

    def limiter(self, x):
        return 1 + math.atan(x - 1)

    def propose_step(self, error):
        inv_error = 1 / (float(error) + self.eps)
        if not self.errs:
            self.errs = [inv_error, inv_error, inv_error]
        self.errs[0] = inv_error
        factor = self.errs[0] ** self.b1 * self.errs[1] ** self.b2 * self.errs[2] ** self.b3
        factor = self.limiter(factor)
        accept = factor >= self.accept_safety
        if accept:
            self.errs[2] = self.errs[1]
            self.errs[1] = self.errs[0]
        self.h *= factor
        return accept


def _dpm_t(sigma):
    """t = -log(sigma) as the reference computes it: an fp32 tensor op (DPMSolver.t, sampling.py:343-344)."""
    return float(-torch.tensor(float(sigma)).log())


def _dpm_sigma(t):
    return math.exp(-t)


def _dpm_eps_op(dst, x_name, den_name, sigma):
    """eps = (x - den) / sigma as one lincomb (DPMSolver.eps, sampling.py:350-357)"""
    return ('lin', dst, [(x_name, 1 / sigma), (den_name, -1 / sigma)])


def _dpm_step_ops(t, t_next, order, dst, r1=None):
    """DPM-Solver step of order 1 / 2 / 3 from t to t_next (sampling.py:359-388) as lincombs over x, eps = (x - D(x, sigma(t))) / sigma(t)
    (already in 'eps') and the intermediate states -- the reference's own association: combining x with u1 / u2 directly would
    cancel ~13 |x| at sigma 80 and lose three digits.
      order 1:  x - A eps
      order 2:  u1 = x - B eps;  x - (A - C) eps - C eps_r1
      order 3:  u1 = x - B1 eps;  u2 = x - (B2 - D2) eps - D2 eps_r1;  x - (A - E) eps - E eps_r2
    Returns (ops, sigmas of the EXTRA evaluations)."""
    h = t_next - t
    sn = _dpm_sigma(t_next)
    A = sn * math.expm1(h)
    if order == 1:
        return [('lin', dst, [('x', 1.), ('eps', -A)])], []
    if order == 2:
        r1 = 1 / 2 if r1 is None else r1
        s1s = _dpm_sigma(t + r1 * h)
        B = s1s * math.expm1(r1 * h)
        C = sn / (2 * r1) * math.expm1(h)
        return [('lin', 'u1', [('x', 1.), ('eps', -B)]), ('eval', 'den1', 'u1'), _dpm_eps_op('eps1', 'u1', 'den1', s1s),
                ('lin', dst, [('x', 1.), ('eps', -(A - C)), ('eps1', -C)])], [s1s]
    r1, r2 = 1 / 3, 2 / 3
    s1s, s2s = _dpm_sigma(t + r1 * h), _dpm_sigma(t + r2 * h)
    B1 = s1s * math.expm1(r1 * h)
    B2 = s2s * math.expm1(r2 * h)
    D2 = s2s * (r2 / r1) * (math.expm1(r2 * h) / (r2 * h) - 1)
    E = sn / r2 * (math.expm1(h) / h - 1)
    return [('lin', 'u1', [('x', 1.), ('eps', -B1)]), ('eval', 'den1', 'u1'), _dpm_eps_op('eps1', 'u1', 'den1', s1s),
            ('lin', 'u2', [('x', 1.), ('eps', -(B2 - D2)), ('eps1', -D2)]), ('eval', 'den2', 'u2'), _dpm_eps_op('eps2', 'u2', 'den2', s2s),
            ('lin', dst, [('x', 1.), ('eps', -(A - E)), ('eps2', -E)])], [s1s, s2s]


def _dpm_ancestral_target(t, t_next, t_end, eta):
    """(t_next_, su) of the stochastic variants (sampling.py:421-426, :455-460).  sigma_down comes from a cancelling difference of
    squares: it is evaluated with the reference's own fp32 tensor ops (host-side 0-dim tensors) so the shortened step matches bit for bit."""
    if not eta:
        return t_next, 0.
    T = lambda v: torch.tensor(float(v), dtype=torch.float32)
    sig = lambda u: u.neg().exp()
    sd, _ = get_ancestral_step(sig(T(t)), sig(T(t_next)), eta)
    t_down = torch.minimum(T(t_end), -sd.log())
    su = (sig(T(t_next)) ** 2 - sig(t_down) ** 2) ** 0.5
    return float(t_down), float(su)


def plan_dpm_fast(sigma_min, sigma_max, n, eta=0., s_noise=1., t_range=None):
    """Host plan of dpm_solver_fast (sampling.py:403-433): (plan, ts) with ts the fp32 time grid as Python floats.  `t_range` =
    (t_start, t_end) gives the end points directly (DPMSolver.dpm_solver_fast is called with times, not sigmas)."""
    if sigma_min <= 0 or sigma_max <= 0:
        raise ValueError('sigma_min and sigma_max must not be 0')
    m = math.floor(n / 3) + 1
    t_lo, t_hi = (-torch.tensor(float(sigma_max)).log(), -torch.tensor(float(sigma_min)).log()) if t_range is None else \
                 (torch.tensor(float(t_range[0])), torch.tensor(float(t_range[1])))
    ts = [float(v) for v in torch.linspace(t_lo, t_hi, m + 1)]
    orders = [3] * (m - 2) + [2, 1] if n % 3 == 0 else [3] * (m - 1) + [n % 3]
    plan = []
    for i, order in enumerate(orders):
        t, t_next = ts[i], ts[i + 1]
        t_down, su = _dpm_ancestral_target(t, t_next, ts[-1], eta)
        ops, extra = _dpm_step_ops(t, t_down, order, 'x')
        ops = [('eval', 'den', 'x'), _dpm_eps_op('eps', 'x', 'den', _dpm_sigma(t))] + ops
        if eta:
            ops += [('noise', 'n', _dpm_sigma(t), _dpm_sigma(t_next)), ('lin', 'x', [('x', 1.), ('n', su * s_noise)])]
        plan.append(dict(i=i, sigma_hat=_dpm_sigma(t), t=t, ops=ops, evals=[_dpm_sigma(t)] + extra))
    return plan, ts


@_on_x_device
@torch.no_grad()
def sample_dpm_fast(model, x, sigma_min, sigma_max, n, extra_args=None, callback=None, disable=None, eta=0., s_noise=1., noise_sampler=None,
                    _t_range=None, _on_eval=None):
    """DPM-Solver-Fast (fixed step size). See https://arxiv.org/abs/2206.00927.  (reference sampling.py:491-501)
    With eta = 0 no noise is drawn at all (the reference draws and multiplies by 0: same samples, different global RNG offset)."""
    plan, ts = plan_dpm_fast(sigma_min, sigma_max, n, eta, s_noise, _t_range)
    sigmas = torch.tensor([_dpm_sigma(t) for t in ts], dtype=torch.float32, device=x.device)
    if eta and noise_sampler is None:
        noise_sampler = default_noise_sampler(_native.f32c(x))
    extra = lambda st: {'t': _scalar_like(sigmas, st['t']), 't_up': _scalar_like(sigmas, st['t'])}
    return _sample_ops('dpm_fast', model, x, sigmas, plan, extra_args, callback, disable, (float(sigma_min), float(sigma_max), n, eta, s_noise),
                       noise_sampler if eta else None, callback_extra=extra, on_eval=_on_eval)


@_on_x_device
@torch.no_grad()
def sample_dpm_adaptive(model, x, sigma_min, sigma_max, extra_args=None, callback=None, disable=None, order=3, rtol=0.05, atol=0.0078, h_init=0.05,
                        pcoeff=0., icoeff=1., dcoeff=0., accept_safety=0.81, eta=0., s_noise=1., noise_sampler=None, return_info=False,
                        _t_range=None, _on_eval=None):
    """DPM-Solver-12 and 23 (adaptive step size). See https://arxiv.org/abs/2206.00927.  (reference sampling.py:435-488, :504-516)
    The step size depends on the data: every step reads one error norm back to the host (`kdb_solver_dpm_error`), so this sampler is
    not captured into a CUDA graph.  Model evaluations, state updates and the error reduction are libkdb200 kernels."""
    if sigma_min <= 0 or sigma_max <= 0:
        raise ValueError('sigma_min and sigma_max must not be 0')
    if order not in {2, 3}:
        raise ValueError('order should be 2 or 3')
    _native.require_cuda(x)
    extra_args = {} if extra_args is None else extra_args
    xc = _native.f32c(x)
    ours = isinstance(noise_sampler, (BrownianTreeNoiseSampler, PhiloxNoiseSampler))
    if eta and noise_sampler is None:
        noise_sampler, ours = default_noise_sampler(xc), True
    t_start, t_end = (f32(_dpm_t(sigma_max)), f32(_dpm_t(sigma_min))) if _t_range is None else (f32(_t_range[0]), f32(_t_range[1]))
    on_eval = (lambda: None) if _on_eval is None else _on_eval
    pid = PIDStepSizeController(abs(h_init), pcoeff, icoeff, dcoeff, 1.5 if eta else order, accept_safety)
    s, x_prev = t_start, xc
    info = {'steps': 0, 'nfe': 0, 'n_accept': 0, 'n_reject': 0}
    while s < f32(t_end - f32(1e-5)):                     # (the reference's s and t are fp32 tensors: same roundings here)
        t = min(t_end, f32(s + f32(pid.h)))
        t_down, su = _dpm_ancestral_target(float(s), float(t), float(t_end), eta)
        if order == 2:
            lo_ops, _ = _dpm_step_ops(float(s), t_down, 1, 'lo')
            hi_ops, evals = _dpm_step_ops(float(s), t_down, 2, 'hi')
            ops = lo_ops + hi_ops
        else:                                              # the order-2 estimate reuses the order-3 step's first stage (same eps_r1 cache key)
            hi_ops, evals = _dpm_step_ops(float(s), t_down, 3, 'hi')
            lo_ops, _ = _dpm_step_ops(float(s), t_down, 2, 'lo', r1=1 / 3)
            ops = hi_ops[:3] + [lo_ops[3]] + hi_ops[3:]      # u1, den1, eps1 | lo | u2, den2, eps2, hi
        ev = _Evaluator(model, xc, extra_args, [_dpm_sigma(float(s))] + evals)
        T, k = {'x': xc}, 0
        for op in [('eval', 'den', 'x'), _dpm_eps_op('eps', 'x', 'den', _dpm_sigma(float(s)))] + ops:
            k += _exec_op(op, T, ev, k)
            if op[0] == 'eval':
                on_eval()
        error = _native.dpm_error(T['lo'], T['hi'], x_prev, atol, rtol)
        accept = pid.propose_step(error)
        if accept:
            x_prev = T['lo']
            xc = T['hi']
            if eta:
                args = (_dpm_sigma(float(s)), _dpm_sigma(float(t))) if ours else (_scalar_like(xc, _dpm_sigma(float(s))), _scalar_like(xc, _dpm_sigma(float(t))))
                xc = _native.lincomb([xc, _native.f32c(noise_sampler(*args))], [1., su * s_noise])
            s = t
            info['n_accept'] += 1
        else:
            info['n_reject'] += 1
        info['nfe'] += order
        info['steps'] += 1
        if callback is not None:
            sg = _scalar_like(xc, _dpm_sigma(float(s)))
            callback({'sigma': sg, 'sigma_hat': sg, 'x': xc, 'i': info['steps'] - 1, 't': _scalar_like(xc, float(s)), 't_up': _scalar_like(xc, float(s)),
                      'denoised': T['den'], 'error': error, 'h': pid.h, **info})
    out = _finish(xc, x)
    return (out, info) if return_info else out


class DPMSolver:
    """DPM-Solver. See https://arxiv.org/abs/2206.00927.  The reference's driver object (sampling.py:333-488) with its constructor and
    its two entry points; times are t = -log(sigma).  The step formulas themselves are the op plans above (`_dpm_step_ops`), so the
    reference's `dpm_solver_{1,2,3}_step` / `eps` cache methods have no counterpart here.  Forward (denoising) direction only."""

    def __init__(self, model, extra_args=None, eps_callback=None, info_callback=None):
        self.model = model
        self.extra_args = {} if extra_args is None else extra_args
        self.eps_callback = eps_callback          # called after every model evaluation
        self.info_callback = info_callback        # called once per step with {'x', 'i', 't', 't_up', 'denoised', ...}

    def t(self, sigma):
        return -sigma.log()

    def sigma(self, t):
        return t.neg().exp()

    @staticmethod
    def _range(t_start, t_end, eta):
        t_start, t_end = float(t_start), float(t_end)
        if not t_end > t_start:
            if eta:
                raise ValueError('eta must be 0 for reverse sampling')
            raise NotImplementedError('reverse-time integration (t_end < t_start) is outside the sampling path of this package')
        return t_start, t_end

    def dpm_solver_fast(self, x, t_start, t_end, nfe, eta=0., s_noise=1., noise_sampler=None):
        t_start, t_end = self._range(t_start, t_end, eta)
        return sample_dpm_fast(self.model, x, math.exp(-t_end), math.exp(-t_start), nfe, extra_args=self.extra_args, callback=self.info_callback,
                               disable=True, eta=eta, s_noise=s_noise, noise_sampler=noise_sampler, _t_range=(t_start, t_end),
                               _on_eval=self.eps_callback)

    def dpm_solver_adaptive(self, x, t_start, t_end, order=3, rtol=0.05, atol=0.0078, h_init=0.05, pcoeff=0., icoeff=1., dcoeff=0.,
                            accept_safety=0.81, eta=0., s_noise=1., noise_sampler=None):
        t_start, t_end = self._range(t_start, t_end, eta)
        return sample_dpm_adaptive(self.model, x, math.exp(-t_end), math.exp(-t_start), extra_args=self.extra_args, callback=self.info_callback,
                                   disable=True, order=order, rtol=rtol, atol=atol, h_init=h_init, pcoeff=pcoeff, icoeff=icoeff, dcoeff=dcoeff,
                                   accept_safety=accept_safety, eta=eta, s_noise=s_noise, noise_sampler=noise_sampler, return_info=True,
                                   _t_range=(t_start, t_end), _on_eval=self.eps_callback)


# --------------------------------------------------------------------------------------------
# log-likelihood by the probability-flow ODE (SURVEY 8f.4; reference sampling.py:280-301)
# --------------------------------------------------------------------------------------------

# Dormand-Prince 5(4), Shampine's error weights and mid-point weights: the method behind torchdiffeq's `method='dopri5'`, which the
# reference calls (sampling.py:298).  torchdiffeq is not part of the reference tree, so its accept / reject sequence cannot be pinned;
# the integrated value is (tests: closed form for Gaussian data, and the oracle's autograd evaluation of the same ODE).
_DP5_ALPHA = (1 / 5, 3 / 10, 4 / 5, 8 / 9, 1., 1.)
_DP5_BETA = ((1 / 5,),
             (3 / 40, 9 / 40),
             (44 / 45, -56 / 15, 32 / 9),
             (19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729),
             (9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656),
             (35 / 384, 0., 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84))
_DP5_C_ERR = (35 / 384 - 1951 / 21600, 0., 500 / 1113 - 22642 / 50085, 125 / 192 - 451 / 720, -2187 / 6784 + 12231 / 42400,
              11 / 84 - 649 / 6300, -1 / 60)
_DP5_C_MID = (6025192743 / 30085553152 / 2, 0., 51252292925 / 65400821598 / 2, -2691868925 / 45128329728 / 2,
              187940372067 / 1594534317056 / 2, -1776094331 / 19743644256 / 2, 11237099 / 235043384 / 2)


def _lin_x(terms, keep_zero=False):
    """sum_i c_i t_i over image-sized tensors: libkdb200 lincomb launches of at most six inputs each"""
    terms = [(t, float(c)) for t, c in terms if keep_zero or c != 0.]
    acc = _native.lincomb([t for t, _ in terms[:6]], [c for _, c in terms[:6]])
    for i in range(6, len(terms), 5):
        part = terms[i:i + 5]
        acc = _native.lincomb([acc] + [t for t, _ in part], [1.] + [c for _, c in part])
    return acc


def _lin_pair(y, h, ks, cs):
    """y + h * sum_j cs[j] * ks[j] for the (latent, ll) pair of the likelihood ODE (y = None: the sum alone); ll is a [B] vector"""
    x_new = _lin_x(([(y[0], 1.)] if y is not None else []) + [(k[0], h * c) for k, c in zip(ks, cs)])
    ll_new = sum(k[1] * (h * c) for k, c in zip(ks, cs) if c != 0.)
    return x_new, (ll_new if y is None else y[1] + ll_new)


def _rk_ratio(err, y0, y1, atol, rtol):
    """max over the two members of the state of rms(err / (atol + rtol max(|y0|, |y1|))): one device->host read"""
    rx = _native.rk_error(err[0], y0[0], y1[0], atol, rtol)
    rl = (err[1] / (atol + rtol * torch.maximum(y0[1].abs(), y1[1].abs()))).pow(2).mean().sqrt()
    return max(rx, float(rl))


def _odeint_dopri5(func, y0, t0, t1, atol, rtol, safety=0.9, ifactor=10., dfactor=0.2, max_steps=100000):
    """y(t1) of dy/dt = func(t, y), y(t0) = y0, for the (latent, log-likelihood change) pair.  Adaptive steps decided on the host from
    one error ratio per step; the step that crosses t1 is evaluated there by the 4th-order dense output (no step is clipped)."""
    f0 = func(t0, y0)
    # first step (Hairer, Norsett & Wanner II.4) with the order of the embedded estimate, 4
    norm = lambda v, ref: _rk_ratio(v, ref, ref, atol, rtol)          # rms(v / (atol + rtol |ref|)), the larger member
    d0, d1 = norm(y0, y0), norm(f0, y0)
    h0 = 1e-6 if d0 < 1e-5 or d1 < 1e-5 else 0.01 * d0 / d1
    f1 = func(t0 + h0, _lin_pair(y0, h0, [f0], [1.]))
    d2 = norm(_lin_pair(None, 1., [f1, f0], [1., -1.]), y0) / h0
    h1 = max(1e-6, h0 * 1e-3) if d1 <= 1e-15 and d2 <= 1e-15 else (0.01 / max(d1, d2)) ** (1 / 5)
    dt = min(100 * h0, h1)
    stats = {'n_accept': 0, 'n_reject': 0}
    t, y = t0, y0
    for _ in range(max_steps):
        ks = [f0]
        for a, row in zip(_DP5_ALPHA, _DP5_BETA):
            y_stage = _lin_pair(y, dt, ks, row)
            ks.append(func(t + a * dt, y_stage))
        y1 = y_stage                                           # the 7th stage point IS the 5th-order solution (first same as last)
        err = _lin_pair(None, dt, ks, _DP5_C_ERR)
        ratio = _rk_ratio(err, y, y1, atol, rtol)
        if not math.isfinite(ratio):
            raise FloatingPointError('log_likelihood: non-finite error estimate')
        factor = ifactor if ratio == 0 else min(ifactor, max(safety / ratio ** (1 / 5), 1. if ratio < 1 else dfactor))
        if ratio <= 1:
            stats['n_accept'] += 1
            if t + dt >= t1:
                y_mid = _lin_pair(y, dt, ks, _DP5_C_MID)
                u = (t1 - t) / dt
                u2, u3, u4 = u * u, u ** 3, u ** 4
                cs = (-8 * u4 + 18 * u3 - 11 * u2 + 1, -8 * u4 + 14 * u3 - 5 * u2, 16 * u4 - 32 * u3 + 16 * u2,
                      dt * (-2 * u4 + 5 * u3 - 4 * u2 + u), dt * (2 * u4 - 3 * u3 + u2))
                members = (y, y1, y_mid, f0, ks[6])
                out_x = _lin_x([(m[0], c) for m, c in zip(members, cs)])
                out_ll = sum(m[1] * c for m, c in zip(members, cs))
                return (out_x, out_ll), stats
            t, y, f0 = t + dt, y1, ks[6]
        else:
            stats['n_reject'] += 1
        dt *= factor
    raise RuntimeError('log_likelihood: max_steps exceeded')


def _likelihood_rhs(model, x, extra_args, v, fd_eps, jvp=False):
    """func(sigma, (x, ll)) -> (d, d_ll) of the likelihood ODE, d = (x - D(x, sigma)) / sigma, d_ll = v^T (dd/dx) v; plus the call counter."""
    from .layers import Denoiser
    B = x.shape[0]
    vv = (v * v).flatten(1).sum(1)
    native = isinstance(model, Denoiser) and model.is_native() and set(extra_args) <= _NATIVE_KW
    count = [0]

    def rhs_native(sigma, y):
        xs = y[0]
        e = fd_eps * math.sqrt(sigma * sigma + float(model.sigma_data) ** 2)
        ev = _Evaluator(model, xs, extra_args, [sigma] * 5)
        ev.precision = _native.PREC_FP32                          # differences of bf16 outputs carry no derivative information
        den = ev(0, xs)
        p1, m1, p2, m2 = (ev(1 + j, _native.lincomb([xs, v], [1., c * e])) for j, c in enumerate((1., -1., 2., -2.)))
        count[0] += 1
        jv = _native.lincomb([p1, m1, p2, m2], [8 / (12 * e), -8 / (12 * e), -1 / (12 * e), 1 / (12 * e)])     # J_D v + O(e^4)
        quad = (v * jv).flatten(1).sum(1)                                                                      # v^T J_D v
        return _native.lincomb([xs, den], [1. / sigma, -1. / sigma]), (vv - quad) / sigma

    def rhs_jvp(sigma, y):
        xs = y[0]
        den, jv = _Evaluator(model, xs, extra_args, [sigma]).jvp(0, xs, v)       # exact J_D v, one engine call
        count[0] += 1
        quad = (v * jv).flatten(1).sum(1)
        return _native.lincomb([xs, den], [1. / sigma, -1. / sigma]), (vv - quad) / sigma

    def rhs_autograd(sigma, y):
        with torch.enable_grad():
            xs = y[0].detach().requires_grad_()
            denoised = model(xs, xs.new_full([B], sigma), **extra_args)
            if not denoised.requires_grad:
                raise RuntimeError('log_likelihood: the model output does not depend on x through torch.autograd; pass a native '
                                   'Denoiser (finite-difference divergence) or a differentiable torch model')
            d = (xs - denoised) / sigma
            count[0] += 1
            grad = torch.autograd.grad((d * v).sum(), xs)[0]
            d_ll = (v * grad).flatten(1).sum(1)
        return _native.f32c(d.detach()), d_ll.detach().float()

    return ((rhs_jvp if jvp else rhs_native) if native else rhs_autograd), count


@_on_x_device
@torch.no_grad()
def log_likelihood(model, x, sigma_min, sigma_max, extra_args=None, atol=1e-4, rtol=1e-4, *, v=None, fd_eps=1e-2, jvp=False):
    """log p(x) at noise level sigma_min by integrating the probability-flow ODE to sigma_max with the Hutchinson estimate
    v^T (dd/dx) v of its divergence, d = (x - D(x, sigma)) / sigma (reference sampling.py:280-301).  Returns (ll [B], {'fevals': n, ...}).

    The quadratic form needs a derivative of the model along v:
      * a native `Denoiser` has forward kernels only, so J_D v is taken as the 4th-order central difference
        (8 (D(x + e v) - D(x - e v)) - (D(x + 2e v) - D(x - 2e v))) / 12e on the exact fp32 path, e = fd_eps * sqrt(sigma^2 + sigma_data^2)
        -- five engine evaluations per ODE function call.  It is the same estimator as the reference's autograd VJP (v^T J v is one
        number, forward or reverse mode); on the cfg1 model it is within 1e-3 absolute of float64 autograd at every sigma (values up to
        784) and the integrated log-likelihood agrees to 6e-6 relative at tight tolerances.
        With `jvp=True` the engine's forward-mode derivative gives J_D v exactly (up to fp32 rounding) in one fp32 engine call per
        ODE function call instead; `fd_eps` is then unused.
      * any other (torch-differentiable) model goes through torch.autograd exactly as in the reference, whatever `jvp` says.
    At the default tolerances two correct integrations differ by a few rtol * |ll| (the step sequence decides); compare at tighter ones.
    `v` (+-1 per element, default torch.randint_like as in the reference) can be passed so that two implementations share the probe."""
    _native.require_cuda(x)
    extra_args = {} if extra_args is None else extra_args
    xc = _native.f32c(x)
    v = (torch.randint_like(xc, 2) * 2 - 1) if v is None else _native.f32c(v.to(xc.device))
    rhs, count = _likelihood_rhs(model, xc, extra_args, v, fd_eps, jvp)
    y0 = (xc, xc.new_zeros([xc.shape[0]]))
    t0, t1 = (float(f32(s_)) for s_ in (sigma_min, sigma_max))          # (:297) the reference's end points are an fp32 tensor
    (latent, delta_ll), stats = _odeint_dopri5(rhs, y0, t0, t1, atol, rtol)
    ll_prior = torch.distributions.Normal(0, float(sigma_max)).log_prob(latent).flatten(1).sum(1)
    return ll_prior + delta_ll, {'fevals': count[0], **stats}
