"""Karras et al. preconditioner (reference: k_diffusion/layers.py:45-90) on native kernels."""
import torch
from torch import nn

from . import _native, utils


class Denoiser(nn.Module):
    """D(x, sigma) = c_skip x + c_out F(c_in x, sigma).

    With an `ImageTransformerDenoiserModelV2` inside, the three scalings are folded into the
    engine's first and last kernels; any other `inner_model` is wrapped with two elementwise
    kernels (scale-in, combine).  `loss` trains an `ImageTransformerDenoiserModelV2` or an
    `ImageDenoiserModelV1` U-Net on its native engine (parameter gradients) and any other inner
    model through torch autograd.
    """

    def __init__(self, inner_model, sigma_data=1., weighting='karras', scales=1):
        super().__init__()
        self.inner_model = inner_model
        self.sigma_data = sigma_data
        self.scales = scales
        named = {'karras': torch.ones_like, 'soft-min-snr': self._weighting_soft_min_snr, 'snr': self._weighting_snr}
        if callable(weighting):
            self.weighting = weighting
        elif weighting in named:
            self.weighting = named[weighting]
        else:
            raise ValueError(f'Unknown weighting type {weighting}')

    def _weighting_soft_min_snr(self, sigma):
        return (sigma * self.sigma_data) ** 2 / (sigma ** 2 + self.sigma_data ** 2) ** 2

    def _weighting_snr(self, sigma):
        return self.sigma_data ** 2 / (sigma ** 2 + self.sigma_data ** 2)

    def get_scalings(self, sigma):
        var = sigma ** 2 + self.sigma_data ** 2
        return self.sigma_data ** 2 / var, sigma * self.sigma_data / var ** 0.5, 1 / var ** 0.5

    _loss_kind = _native.LOSS_DENOISER

    def _check_loss(self):
        if self.scales != 1:
            raise NotImplementedError('loss with scales != 1 weights the error by frequency through a DCT (dctorch), which is not built')

    def loss(self, input, noise, sigma, **kwargs):
        """Per-sample losses [B] (reference layers.py:76-86, scales == 1).  A native image_transformer_v2 inner model runs one fp32 engine
        evaluation and one loss kernel, and its backward one native call that writes every parameter's gradient; the image_v1 U-Net does the
        same at exact fp32; image_transformer_v1 raises NotImplementedError.  Any other inner model runs the reference formula under torch
        autograd.

        A native inner model wrapped in torch.nn.parallel.DistributedDataParallel (as Accelerate wraps it) runs its native loss inside
        the wrapper's forward, called with the keyword `loss_request`; its backward writes every gradient at once, and DDP's reducer
        averages them across the ranks (or, under no_sync(), leaves them to accumulate).  A model whose loss leaves some parameters
        without a gradient -- a U-Net with skip_stages > 0, or mapping_cond.* when no mapping_cond is formed -- needs
        find_unused_parameters=True, as under torch autograd."""
        self._check_loss()
        inner = utils.unwrap_ddp(self.inner_model)
        native_loss = getattr(inner, 'native_loss', None)
        if native_loss is not None:
            request = _native.LossRequest(self._loss_kind, noise, self.sigma_data, self.weighting(sigma))
            if inner is not self.inner_model:
                # through DistributedDataParallel.forward, which prepares the reducer that all-reduces the backward's gradients
                return self.inner_model(input, sigma, **kwargs, loss_request=request)
            return request(native_loss, input, sigma, **kwargs)
        if self.is_native():
            raise NotImplementedError(f'{type(self.inner_model).__name__}: parameter gradients are built for image_transformer_v2 models only')
        return self._torch_loss(input, noise, sigma, **kwargs)

    def _torch_loss(self, input, noise, sigma, **kwargs):
        c_skip, c_out, c_in = [utils.append_dims(x, input.ndim) for x in self.get_scalings(sigma)]
        c_weight = self.weighting(sigma)
        noised_input = input + noise * utils.append_dims(sigma, input.ndim)
        model_output = self.inner_model(noised_input * c_in, sigma, **kwargs)
        target = (input - c_skip * noised_input) / c_out
        return ((model_output - target) ** 2).flatten(1).mean(1) * c_weight

    def is_native(self):
        """Whether the inner model, seen through a DistributedDataParallel wrapper, has a native front end (`native_eval`), which the
        fused paths here and the samplers evaluate through."""
        return getattr(utils.unwrap_ddp(self.inner_model), 'native_eval', None) is not None

    def forward(self, input, sigma, **kwargs):
        _native.require_cuda(input, sigma)
        if self.is_native():
            return utils.unwrap_ddp(self.inner_model).denoise(input, sigma, self.sigma_data, **kwargs)
        x = _native.f32c(input)
        sig = _native.f32c(sigma).expand(x.shape[0]).contiguous()
        f = self.inner_model(_native.precond_scale_in(x, sig, float(self.sigma_data)), sigma, **kwargs)
        return _native.precond_combine(_native.f32c(f), x, sig, float(self.sigma_data))

    def jvp(self, input, sigma, tangent, **kwargs):
        """(D(x, sigma), J_D(x) tangent): the denoiser and its forward-mode derivative with respect to `input` along `tangent`.

        A native inner model computes both in one fp32 engine call.  Any other inner model goes through `torch.func.jvp` of
        inner(c_in x); the combine c_skip x + c_out f is linear, so one combine kernel serves the primal and the tangent."""
        _native.require_cuda(input, sigma, tangent)
        if self.is_native():
            return utils.unwrap_ddp(self.inner_model).denoise_jvp(input, sigma, tangent, self.sigma_data, **kwargs)
        x, t = _native.f32c(input), _native.f32c(tangent)
        sig = _native.f32c(sigma).expand(x.shape[0]).contiguous()
        sd = float(self.sigma_data)
        c_in = (1 / (sig * sig + sd * sd).sqrt()).view(-1, *([1] * (x.ndim - 1)))
        f, df = torch.func.jvp(lambda xx: self.inner_model(xx * c_in, sigma, **kwargs), (x,), (t,))
        return _native.precond_combine(_native.f32c(f), x, sig, sd), _native.precond_combine(_native.f32c(df), t, sig, sd)

    def vjp(self, input, sigma, cotangent, **kwargs):
        """(D(x, sigma), cotangent^T J_D(x)): the denoiser and its reverse-mode derivative with respect to `input`.

        A native inner model computes both in one fp32 engine call.  Any other inner model goes through `torch.func.vjp` of
        inner(c_in x), whose gradient g = c_in J_F^T u is linear in u, so c_skip u + c_in J_F^T (c_out u) = c_out g + c_skip u is
        one combine kernel, as in `jvp`."""
        _native.require_cuda(input, sigma, cotangent)
        if self.is_native():
            return utils.unwrap_ddp(self.inner_model).denoise_vjp(input, sigma, cotangent, self.sigma_data, **kwargs)
        x, u = _native.f32c(input), _native.f32c(cotangent)
        sig = _native.f32c(sigma).expand(x.shape[0]).contiguous()
        sd = float(self.sigma_data)
        c_in = (1 / (sig * sig + sd * sd).sqrt()).view(-1, *([1] * (x.ndim - 1)))
        f, pull = torch.func.vjp(lambda xx: self.inner_model(xx * c_in, sigma, **kwargs), x)
        (g,) = pull(u.to(f.dtype))
        return _native.precond_combine(_native.f32c(f), x, sig, sd), _native.precond_combine(_native.f32c(g), u, sig, sd)


class DenoiserWithVariance(Denoiser):
    """reference layers.py:93-101: differs from Denoiser in `loss` only, which needs the inner model's learned variance; sampling is
    identical.

    `loss` (scales and weighting are accepted and ignored, as in the reference) runs natively around an image_v1 U-Net with has_variance,
    bare, in KarrasAugmentWrapper or in DistributedDataParallel: one fp32 engine evaluation that also forms logvar, one loss kernel, and a
    backward that writes every parameter's gradient, proj_out's variance row included.  The transformers and a U-Net without has_variance
    raise NotImplementedError; any other inner model runs the reference formula under torch autograd, called with return_variance=True."""

    _loss_kind = _native.LOSS_VARIANCE

    def _check_loss(self):
        pass

    def _torch_loss(self, input, noise, sigma, **kwargs):
        c_skip, c_out, c_in = [utils.append_dims(x, input.ndim) for x in self.get_scalings(sigma)]
        noised_input = input + noise * utils.append_dims(sigma, input.ndim)
        model_output, logvar = self.inner_model(noised_input * c_in, sigma, return_variance=True, **kwargs)
        logvar = utils.append_dims(logvar, model_output.ndim)
        target = (input - c_skip * noised_input) / c_out
        losses = ((model_output - target) ** 2 / logvar.exp() + logvar) / 2
        return losses.flatten(1).mean(1)


class SimpleLossDenoiser(Denoiser):
    """L_simple with the Karras et al. preconditioner (reference layers.py:104-113): differs from Denoiser in `loss` only."""

    _loss_kind = _native.LOSS_SIMPLE

    def _torch_loss(self, input, noise, sigma, **kwargs):
        c_skip, c_out, c_in = [utils.append_dims(x, input.ndim) for x in self.get_scalings(sigma)]
        noised_input = input + noise * utils.append_dims(sigma, input.ndim)
        denoised = self.inner_model(noised_input * c_in, sigma, **kwargs) * c_out + noised_input * c_skip
        eps = (noised_input - denoised) / utils.append_dims(sigma, input.ndim)
        return (eps - noise).pow(2).flatten(1).mean(1)


class FourierFeatures(nn.Module):
    """Random Fourier features buffer (layers.py:285-293); evaluated inside the engine's conditioning kernel."""

    def __init__(self, in_features, out_features, std=1.):
        super().__init__()
        assert out_features % 2 == 0
        self.register_buffer('weight', torch.randn([out_features // 2, in_features]) * std)
