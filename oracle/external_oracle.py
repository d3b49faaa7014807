"""Torch restatement of the reference's external model wrappers (k_diffusion/external.py:9-38, 87-177).  TEST INFRASTRUCTURE ONLY.

Each wrapper's forward is written out op for op in the order the reference evaluates it, so on a given device it rounds exactly as
the reference does: tests/test_external_host.py holds it to the reference's outputs recorded by oracle/make_golden_external.py, and
tests/test_gpu_external.py holds the native wrappers to it, run by torch on the same GPU.

The toy inner models below are the deterministic eps, v and learned-variance models the fixtures were recorded with.  They are plain
torch modules with one parameter each, so gradients with respect to an inner parameter can be compared too.
"""
import math

import torch
from torch import nn

from .kdiff_oracle import DiscreteScheduleOracle, _bcast


def sd_alphas_cumprod(n=1000, beta_start=0.00085, beta_end=0.012):
    """Stable Diffusion's ("scaled linear") schedule: betas linear in sqrt(beta) from 0.00085 to 0.012 over 1000 steps."""
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    return torch.cumprod(1 - betas, 0)


# ----------------------------------------------------------------------------------------------
# the wrappers (external.py)
# ----------------------------------------------------------------------------------------------

def v_scalings(sigma, sigma_data):
    """external.py:17-21 and 145-149 (c_skip, c_out, c_in)"""
    c_skip = sigma_data ** 2 / (sigma ** 2 + sigma_data ** 2)
    c_out = -sigma * sigma_data / (sigma ** 2 + sigma_data ** 2) ** 0.5
    c_in = 1 / (sigma ** 2 + sigma_data ** 2) ** 0.5
    return c_skip, c_out, c_in


def eps_scalings(sigma, sigma_data):
    """external.py:96-99 (c_out, c_in)"""
    return -sigma, 1 / (sigma ** 2 + sigma_data ** 2) ** 0.5


def v_forward(get_v, t, x, sigma, sigma_data, **kw):
    """external.py:36-38 and 161-163: get_v(c_in x, t, **kw) * c_out + x * c_skip"""
    c_skip, c_out, c_in = [_bcast(c, x.ndim) for c in v_scalings(sigma, sigma_data)]
    return get_v(x * c_in, t, **kw) * c_out + x * c_skip


def eps_forward(get_eps, t, x, sigma, sigma_data, **kw):
    """external.py:110-113: x + get_eps(c_in x, t, **kw) * c_out"""
    c_out, c_in = [_bcast(c, x.ndim) for c in eps_scalings(sigma, sigma_data)]
    return x + get_eps(x * c_in, t, **kw) * c_out


class VDenoiserOracle:
    """external.py:9-38"""

    def __init__(self, inner_model):
        self.inner_model, self.sigma_data = inner_model, 1.0

    def sigma_to_t(self, sigma):
        return sigma.atan() / math.pi * 2

    def t_to_sigma(self, t):
        return (t * math.pi / 2).tan()

    def __call__(self, x, sigma, **kw):
        return v_forward(self.inner_model, self.sigma_to_t(sigma), x, sigma, self.sigma_data, **kw)


class DiscreteEpsDDPMDenoiserOracle(DiscreteScheduleOracle):
    """external.py:87-113"""

    def __init__(self, model, alphas_cumprod, quantize):
        super().__init__(((1 - alphas_cumprod) / alphas_cumprod) ** 0.5, quantize)
        self.inner_model, self.sigma_data = model, 1.0

    def get_eps(self, *args, **kw):
        return self.inner_model(*args, **kw)

    def __call__(self, x, sigma, **kw):
        return eps_forward(self.get_eps, self.sigma_to_t(sigma), x, sigma, self.sigma_data, **kw)


class OpenAIDenoiserOracle(DiscreteEpsDDPMDenoiserOracle):
    """external.py:116-129"""

    def __init__(self, model, diffusion, quantize=False, has_learned_sigmas=True, device="cpu"):
        super().__init__(model, torch.tensor(diffusion.alphas_cumprod, device=device, dtype=torch.float32), quantize)
        self.has_learned_sigmas = has_learned_sigmas

    def get_eps(self, *args, **kw):
        out = self.inner_model(*args, **kw)
        return out.chunk(2, dim=1)[0] if self.has_learned_sigmas else out


class CompVisDenoiserOracle(DiscreteEpsDDPMDenoiserOracle):
    """external.py:132-139"""

    def __init__(self, model, quantize=False, device="cpu"):
        super().__init__(model, model.alphas_cumprod, quantize)

    def get_eps(self, *args, **kw):
        return self.inner_model.apply_model(*args, **kw)


class DiscreteVDDPMDenoiserOracle(DiscreteScheduleOracle):
    """external.py:142-163"""

    def __init__(self, model, alphas_cumprod, quantize):
        super().__init__(((1 - alphas_cumprod) / alphas_cumprod) ** 0.5, quantize)
        self.inner_model, self.sigma_data = model, 1.0

    def get_v(self, *args, **kw):
        return self.inner_model(*args, **kw)

    def __call__(self, x, sigma, **kw):
        return v_forward(self.get_v, self.sigma_to_t(sigma), x, sigma, self.sigma_data, **kw)


class CompVisVDenoiserOracle(DiscreteVDDPMDenoiserOracle):
    """external.py:166-173 (get_v drops its **kwargs)"""

    def __init__(self, model, quantize=False, device="cpu"):
        super().__init__(model, model.alphas_cumprod, quantize)

    def get_v(self, x, t, cond, **kw):
        return self.inner_model.apply_model(x, t, cond)


# ----------------------------------------------------------------------------------------------
# deterministic toy inner models
# ----------------------------------------------------------------------------------------------

class ToyModel(nn.Module):
    """F(x, t) = tanh(w_c x) + 0.3 sin(t / t_scale) (+ 0.1 cond), w one weight per channel.  With `learned_sigmas` the output has
    twice the channels, a second half that must never reach the result; `out_dtype` is the dtype the model returns (Stable Diffusion
    runs in fp16)."""

    def __init__(self, channels, t_scale=1000.0, learned_sigmas=False, out_dtype=torch.float32):
        super().__init__()
        self.weight = nn.Parameter(torch.linspace(0.6, 1.4, channels))
        self.t_scale, self.learned_sigmas, self.out_dtype = t_scale, learned_sigmas, out_dtype

    def forward(self, x, t, cond=None):
        out = torch.tanh(x * self.weight[:, None, None]) + 0.3 * torch.sin(t.float() / self.t_scale)[:, None, None, None]
        if cond is not None:
            out = out + 0.1 * cond
        if self.learned_sigmas:
            out = torch.cat([out, 5.0 + x.flip(1)], dim=1)
        return out.to(self.out_dtype)


class ToyCompVis(nn.Module):
    """A CompVis-style latent diffusion model: `alphas_cumprod` attribute and `apply_model(x, t, cond)`."""

    def __init__(self, channels, out_dtype=torch.float32, alphas_cumprod=None):
        super().__init__()
        self.model = ToyModel(channels, out_dtype=out_dtype)
        self.register_buffer("alphas_cumprod", sd_alphas_cumprod() if alphas_cumprod is None else alphas_cumprod)

    def apply_model(self, x, t, cond):
        return self.model(x, t, cond)


class ToyDiffusion:
    """What OpenAIDenoiser reads of a guided-diffusion GaussianDiffusion: `alphas_cumprod` as a float64 numpy array."""

    def __init__(self, n=1000):
        betas = torch.linspace(0.0001, 0.02, n, dtype=torch.float64)      # guided-diffusion's linear schedule
        self.alphas_cumprod = torch.cumprod(1 - betas, 0).numpy()
