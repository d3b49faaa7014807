"""Wrappers that drive foreign eps- and v-prediction models with the samplers (reference: k_diffusion/external.py).

The discrete noise-level tables (`DiscreteSchedule`, `sigma_to_t`, `t_to_sigma`) are O(table) one-dimensional torch ops on
whatever device the table lives on; they are issued in the same order as the reference so `sigma_to_t` indices are
bit-identical and the float results match to the last bit on the same device.

The per-evaluation math on the latent -- the input scaling c_in x and the eps or v combine -- runs on two native kernels around
the inner model (kdb_external_scale_in, kdb_external_combine).  They round every operation as the reference's torch expressions
do, so a wrapper's output equals the reference's on the same GPU bit for bit.  The inner model's output is read in place, in
fp32, fp16 or bf16, including the eps half of a learned-variance output.  Both kernels sit in autograd Functions with a
backward and a jvp, so guidance, `log_likelihood` and `torch.func.jvp` reach the input and the inner model's parameters.
"""
import math

import torch
from torch import nn
from torch.autograd import forward_ad

from . import _native, sampling


class DiscreteSchedule(nn.Module):
    """A mapping between continuous noise levels (sigmas) and a list of discrete noise levels."""

    def __init__(self, sigmas, quantize):
        super().__init__()
        self.register_buffer('sigmas', sigmas)
        self.register_buffer('log_sigmas', sigmas.log())
        self.quantize = quantize

    @property
    def sigma_min(self):
        return self.sigmas[0]

    @property
    def sigma_max(self):
        return self.sigmas[-1]

    def get_sigmas(self, n=None):
        if n is None:
            return sampling.append_zero(self.sigmas.flip(0))
        last = len(self.sigmas) - 1
        return sampling.append_zero(self.t_to_sigma(torch.linspace(last, 0, n, device=self.sigmas.device)))

    def sigma_to_t(self, sigma, quantize=None):
        if quantize is None:
            quantize = self.quantize
        log_sigma = sigma.log()
        dists = log_sigma - self.log_sigmas[:, None]             # [table, queries]
        if quantize:
            return dists.abs().argmin(dim=0).view(sigma.shape)   # nearest table entry (int64)
        lo_i = dists.ge(0).cumsum(dim=0).argmax(dim=0).clamp(max=self.log_sigmas.shape[0] - 2)
        hi_i = lo_i + 1
        lo, hi = self.log_sigmas[lo_i], self.log_sigmas[hi_i]
        w = ((lo - log_sigma) / (lo - hi)).clamp(0, 1)
        return ((1 - w) * lo_i + w * hi_i).view(sigma.shape)

    def t_to_sigma(self, t):
        t = t.float()
        lo_i, hi_i, w = t.floor().long(), t.ceil().long(), t.frac()
        return ((1 - w) * self.log_sigmas[lo_i] + w * self.log_sigmas[hi_i]).exp()


# ---------------------------------------------------------------------------------------------
# the wrappers' latent math as differentiable native ops
# ---------------------------------------------------------------------------------------------

class _ScaleIn(torch.autograd.Function):
    """x * c_in(sigma): linear in x, so its gradient and its tangent are the same op applied to u or dx.  backward and jvp call
    `apply` again rather than the kernel, so that under a torch.func transform the kernel sees unwrapped tensors."""

    @staticmethod
    def forward(x, sigma, sigma_data):
        return _native.external_scale_in(x, sigma, sigma_data)

    @staticmethod
    def setup_context(ctx, inputs, output):
        _, sigma, ctx.sigma_data = inputs
        ctx.save_for_backward(sigma)
        ctx.save_for_forward(sigma)

    @staticmethod
    def backward(ctx, u):
        (sigma,) = ctx.saved_tensors
        return _ScaleIn.apply(_native.f32c(u), sigma, ctx.sigma_data), None, None

    @staticmethod
    def jvp(ctx, dx, _dsigma, _dsigma_data):
        (sigma,) = ctx.saved_tensors
        return _ScaleIn.apply(_native.f32c(dx), sigma, ctx.sigma_data)


class _Combine(torch.autograd.Function):
    """The output combine of one wrapper kind, affine in (x, f):
      eps: x + f * (-sigma)        g_x = u,         g_f = -sigma u
      v:   f * c_out + x * c_skip  g_x = c_skip u,  g_f = c_out u
    x or f may be None, which drops its term: each gradient is the same op with one term dropped, the tangent is the combine of the
    tangents.  As in _ScaleIn, backward and jvp go through `apply`."""

    @staticmethod
    def forward(kind, x, f, sigma, sigma_data):
        return _native.external_combine(kind, f, x, sigma, sigma_data)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.kind, _, f, sigma, ctx.sigma_data = inputs
        ctx.f_dtype = None if f is None else f.dtype
        ctx.save_for_backward(sigma)
        ctx.save_for_forward(sigma)

    @staticmethod
    def backward(ctx, u):
        (sigma,) = ctx.saved_tensors
        u = _native.f32c(u)
        g_x = g_f = None
        if ctx.needs_input_grad[1]:
            g_x = u if ctx.kind == _native.EXTERNAL_EPS else _Combine.apply(ctx.kind, u, None, sigma, ctx.sigma_data)
        if ctx.needs_input_grad[2]:
            g_f = _Combine.apply(ctx.kind, None, u, sigma, ctx.sigma_data).to(ctx.f_dtype)
        return None, g_x, g_f, None, None

    @staticmethod
    def jvp(ctx, _dkind, dx, df, _dsigma, _dsigma_data):
        (sigma,) = ctx.saved_tensors
        if dx is None and df is None:
            return None
        return _Combine.apply(ctx.kind, None if dx is None else _native.f32c(dx), df, sigma, ctx.sigma_data)


def _derivatives_possible():
    """Whether torch can differentiate the call being made: autograd is recording, a torch.func transform is active or a
    forward-mode dual level is open (a dual tensor can exist only inside one)."""
    return (torch.is_grad_enabled() or torch._C._are_functorch_transforms_active()
            or getattr(forward_ad, "_current_level", 0) >= 0)


def _wrapped_forward(kind, wrapper, inner, input, sigma, **kwargs):
    """combine(x, inner(c_in x, sigma_to_t(sigma), **kwargs), sigma): two native launches around the inner model."""
    _native.require_cuda(input, sigma)
    if sigma.requires_grad:
        raise RuntimeError("the external wrappers differentiate with respect to the input and the inner model, not sigma "
                           "(pass sigma.detach())")
    x = _native.f32c(input)
    B = x.shape[0]
    sig = _native.f32c(sigma.reshape(-1))
    if sig.numel() == 1 and B != 1:
        sig = sig.expand(B).contiguous()
    if sig.numel() != B:
        raise ValueError(f"sigma of shape {tuple(sigma.shape)} for a batch of {B}")
    sd = float(wrapper.sigma_data)
    with _native.device_of(x):
        if not _derivatives_possible():           # the samplers' no_grad loop: skip autograd.Function's per-call bookkeeping
            f = inner(_native.external_scale_in(x, sig, sd), wrapper.sigma_to_t(sigma), **kwargs)
            return _native.external_combine(kind, f, x, sig, sd)
        f = inner(_ScaleIn.apply(x, sig, sd), wrapper.sigma_to_t(sigma), **kwargs)
        return _Combine.apply(kind, x, f, sig, sd)


def _v_scalings(sigma, sigma_data):
    """(c_skip, c_out, c_in) of a v-prediction model as torch tensors; the kernels evaluate the same expressions per sample."""
    var = sigma ** 2 + sigma_data ** 2
    return sigma_data ** 2 / var, -sigma * sigma_data / var ** 0.5, 1 / var ** 0.5


def _training_out_of_scope(*args, **kwargs):
    raise NotImplementedError('training losses are out of scope for the H100 sampling path')


class VDenoiser(nn.Module):
    """Wraps a continuous-time v-prediction model (v-diffusion-pytorch), t = atan(sigma) * 2 / pi."""

    def __init__(self, inner_model):
        super().__init__()
        self.inner_model = inner_model
        self.sigma_data = 1.

    def get_scalings(self, sigma):
        return _v_scalings(sigma, self.sigma_data)

    def sigma_to_t(self, sigma):
        return sigma.atan() / math.pi * 2

    def t_to_sigma(self, t):
        return (t * math.pi / 2).tan()

    def loss(self, input, noise, sigma, **kwargs):
        _training_out_of_scope()

    def forward(self, input, sigma, **kwargs):
        return _wrapped_forward(_native.EXTERNAL_V, self, self.inner_model, input, sigma, **kwargs)


class DiscreteEpsDDPMDenoiser(DiscreteSchedule):
    """Wraps a discrete-time DDPM model that predicts the noise eps, given its alphas_cumprod table."""

    def __init__(self, model, alphas_cumprod, quantize):
        super().__init__(((1 - alphas_cumprod) / alphas_cumprod) ** 0.5, quantize)
        self.inner_model = model
        self.sigma_data = 1.

    def get_scalings(self, sigma):
        return -sigma, 1 / (sigma ** 2 + self.sigma_data ** 2) ** 0.5

    def get_eps(self, *args, **kwargs):
        return self.inner_model(*args, **kwargs)

    def loss(self, input, noise, sigma, **kwargs):
        _training_out_of_scope()

    def forward(self, input, sigma, **kwargs):
        return _wrapped_forward(_native.EXTERNAL_EPS, self, self.get_eps, input, sigma, **kwargs)


class OpenAIDenoiser(DiscreteEpsDDPMDenoiser):
    """Wraps a guided-diffusion (OpenAI) model; with learned sigmas its output carries eps in the first half of the channels."""

    def __init__(self, model, diffusion, quantize=False, has_learned_sigmas=True, device='cpu'):
        alphas_cumprod = torch.tensor(diffusion.alphas_cumprod, device=device, dtype=torch.float32)
        super().__init__(model, alphas_cumprod, quantize=quantize)
        self.has_learned_sigmas = has_learned_sigmas

    def get_eps(self, *args, **kwargs):
        model_output = self.inner_model(*args, **kwargs)
        if self.has_learned_sigmas:
            return model_output.chunk(2, dim=1)[0]        # a view: the combine reads it in place with its batch stride
        return model_output


class CompVisDenoiser(DiscreteEpsDDPMDenoiser):
    """Wraps a CompVis latent diffusion (Stable Diffusion) eps model, called through its `apply_model`."""

    def __init__(self, model, quantize=False, device='cpu'):
        super().__init__(model, model.alphas_cumprod, quantize=quantize)

    def get_eps(self, *args, **kwargs):
        return self.inner_model.apply_model(*args, **kwargs)


class DiscreteVDDPMDenoiser(DiscreteSchedule):
    """Wraps a discrete-time DDPM model that predicts v, given its alphas_cumprod table."""

    def __init__(self, model, alphas_cumprod, quantize):
        super().__init__(((1 - alphas_cumprod) / alphas_cumprod) ** 0.5, quantize)
        self.inner_model = model
        self.sigma_data = 1.

    def get_scalings(self, sigma):
        return _v_scalings(sigma, self.sigma_data)

    def get_v(self, *args, **kwargs):
        return self.inner_model(*args, **kwargs)

    def loss(self, input, noise, sigma, **kwargs):
        _training_out_of_scope()

    def forward(self, input, sigma, **kwargs):
        return _wrapped_forward(_native.EXTERNAL_V, self, self.get_v, input, sigma, **kwargs)


class CompVisVDenoiser(DiscreteVDDPMDenoiser):
    """Wraps a CompVis latent diffusion v model (Stable Diffusion 2.x 768-v), called through its `apply_model`."""

    def __init__(self, model, quantize=False, device='cpu'):
        super().__init__(model, model.alphas_cumprod, quantize=quantize)

    def get_v(self, x, t, cond, **kwargs):
        return self.inner_model.apply_model(x, t, cond)       # kwargs are dropped, as in the reference
