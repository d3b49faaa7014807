"""Small helpers on the sampling path (reference: k_diffusion/utils.py:43-48,82-85,429-443) and the pieces of train.py's step that live in
the reference's utils (:88-385, 451-458): the EMA update and its warmup, the learning-rate schedules, stratified uniforms and the sigma
sample densities."""
import math
import threading
import warnings
from contextlib import contextmanager

import torch
from torch import optim


def append_dims(x, target_dims):
    """Right-pad x's shape with singleton dims up to `target_dims` (utils.py:43-48)."""
    extra = target_dims - x.ndim
    if extra < 0:
        raise ValueError(f'input has {x.ndim} dims but target_dims is {target_dims}, which is less')
    return x.reshape(tuple(x.shape) + (1,) * extra)


def to_pil_image(x):
    """[-1, 1] tensor [C,H,W] / [1,C,H,W] -> PIL image (utils.py:27-34): clamp, map to [0, 255] as torchvision's to_pil_image does
    for float input (mul 255, truncate to uint8)."""
    import numpy as np
    from PIL import Image
    if x.ndim == 4:
        assert x.shape[0] == 1
        x = x[0]
    if x.shape[0] == 1:
        x = x[0]
    arr = ((x.detach().float().clamp(-1, 1) + 1) / 2).mul(255).byte().cpu().numpy()
    if arr.ndim == 3:
        arr = np.transpose(arr, (1, 2, 0))
    return Image.fromarray(arr)


def from_pil_image(x):
    """PIL image -> [-1, 1] tensor [C,H,W] (utils.py:19-24)."""
    import numpy as np
    import torch
    arr = np.asarray(x)
    t = torch.from_numpy(arr.copy())
    t = t[None] if t.ndim == 2 else t.permute(2, 0, 1)
    return t.float().div(255) * 2 - 1


def n_params(module):
    return sum(p.numel() for p in module.parameters())


@contextmanager
def _mode(model, training):
    was = [m.training for m in model.modules()]
    try:
        yield model.train(training)
    finally:
        for m, t in zip(model.modules(), was):
            m.training = t


def eval_mode(model):
    """Context manager: put `model` in eval mode, restore on exit (utils.py:82)."""
    return _mode(model, False)


def train_mode(model):
    return _mode(model, True)


@contextmanager
def tf32_mode(cudnn=None, matmul=None):
    """Context manager (and decorator) setting whether cuDNN convolutions and CUDA matmuls may use TF32 (utils.py:429-443).  A flag
    given as True or False is put back to its previous value on exit, also when the body raises; None leaves that flag alone."""
    import torch
    flags = [(torch.backends.cudnn, cudnn), (torch.backends.cuda.matmul, matmul)]
    saved = [owner.allow_tf32 for owner, _ in flags]
    try:
        for owner, value in flags:
            if value is not None:
                owner.allow_tf32 = value
        yield
    finally:
        for (owner, value), old in zip(flags, saved):
            if value is not None:
                owner.allow_tf32 = old


def _ema_pairs(model, averaged_model, named):
    """{name: (averaged tensor, model tensor)} of named_parameters or named_buffers; the key sets must agree (utils.py:92-101)."""
    ours, theirs = dict(getattr(model, named)()), dict(getattr(averaged_model, named)())
    assert ours.keys() == theirs.keys()
    return [(theirs[k], v) for k, v in ours.items()]


def _native_ema_ok(pairs):
    devices = {t.device for pair in pairs for t in pair}
    return (len(devices) == 1 and next(iter(devices)).type == "cuda"
            and all(d.dtype == s.dtype == torch.float32 and d.shape == s.shape and d.is_contiguous() and s.is_contiguous() for d, s in pairs))


@torch.no_grad()
def ema_update(model, averaged_model, decay):
    """Fold the model's parameters into the exponential moving average `averaged_model` (each parameter lerps towards the model's by
    1 - decay) and copy the model's buffers into it; call after each optimizer step (utils.py:88-104).

    When every parameter and buffer pair is a contiguous fp32 tensor on one CUDA device, all of them are updated by one kdb_ema_update
    launch, bit for bit the reference's lerp_ / copy_ on the same GPU; anything else (other dtypes, CPU models, mixed devices) takes the
    reference's per-tensor lerp_ / copy_.  The native write bumps each destination's version counter, as lerp_ and copy_ do, so a native
    engine bound to the averaged model rebinds on its next call."""
    params = _ema_pairs(model, averaged_model, "named_parameters")
    buffers = _ema_pairs(model, averaged_model, "named_buffers")
    weight = 1 - decay
    pairs = params + buffers
    if pairs and _native_ema_ok(pairs):
        from . import _native
        modes = [_native.EMA_LERP] * len(params) + [_native.EMA_COPY] * len(buffers)
        _native.ema_update([d for d, _ in pairs], [s for _, s in pairs], modes, weight)
        torch.autograd.graph.increment_version([d for d, _ in pairs])
        return
    for dst, src in params:
        dst.lerp_(src, weight)
    for dst, src in buffers:
        dst.copy_(src)


def ema_update_dict(values, updates, decay):
    """Exponential moving average of a dict of values (utils.py:451-458): a new key takes its update, a known one decays towards it."""
    for k, v in updates.items():
        if k in values:
            values[k] *= decay
            values[k] += (1 - decay) * v
        else:
            values[k] = v
    return values


class EMAWarmup:
    """EMA decay with an inverse warmup (utils.py:107-152): 1 - (1 + epoch / inv_gamma) ** -power, epoch = steps since `start_at`,
    clamped to [min_value, max_value].  inv_gamma=1, power=2/3 reaches 0.999 at 31.6K steps and 0.9999 at 1M; power=3/4 reaches them at
    10K and 215.4K steps.

    Args:
        inv_gamma (float): Inverse multiplicative factor of EMA warmup. Default: 1.
        power (float): Exponential factor of EMA warmup. Default: 1.
        min_value (float): The minimum EMA decay rate. Default: 0.
        max_value (float): The maximum EMA decay rate. Default: 1.
        start_at (int): The epoch to start averaging at. Default: 0.
        last_epoch (int): The index of last epoch. Default: 0.
    """

    def __init__(self, inv_gamma=1., power=1., min_value=0., max_value=1., start_at=0, last_epoch=0):
        self.inv_gamma, self.power = inv_gamma, power
        self.min_value, self.max_value = min_value, max_value
        self.start_at, self.last_epoch = start_at, last_epoch

    def state_dict(self):
        """The warmup's state as a dict (every attribute)."""
        return dict(self.__dict__)

    def load_state_dict(self, state_dict):
        """Restore a state returned by `state_dict`."""
        self.__dict__.update(state_dict)

    def get_value(self):
        """The current EMA decay rate."""
        epoch = max(0, self.last_epoch - self.start_at)
        value = 1 - (1 + epoch / self.inv_gamma) ** -self.power
        return 0. if epoch < 0 else min(self.max_value, max(self.min_value, value))

    def step(self):
        """Advance one step."""
        self.last_epoch += 1


def _check_warmup(warmup):
    if not 0. <= warmup < 1:
        raise ValueError('Invalid value for warmup')


class _ClosedFormLR(optim.lr_scheduler.LRScheduler):
    """The reference's schedules (utils.py:155-264) compute each learning rate from last_epoch alone; get_lr outside step() warns, as
    torch's own schedulers do.  `verbose` is accepted for the reference's signature; torch no longer takes it."""

    def get_lr(self):
        if not self._get_lr_called_within_step:
            warnings.warn("To get the last learning rate computed by the scheduler, please use `get_last_lr()`.")
        return self._get_closed_form_lr()

    def _warmup(self):
        return 1 - self.warmup ** (self.last_epoch + 1)


class InverseLR(_ClosedFormLR):
    """Inverse decay lr = base_lr (1 + epoch / inv_gamma) ** -power, floored at min_lr, times an exponential warmup 1 - warmup ** (epoch + 1)
    (utils.py:155-193).  inv_gamma is the number of steps for the rate to fall to (1 / 2) ** power of its start.

    Args:
        optimizer (Optimizer): Wrapped optimizer.
        inv_gamma (float): Inverse multiplicative factor of learning rate decay. Default: 1.
        power (float): Exponential factor of learning rate decay. Default: 1.
        warmup (float): Exponential warmup factor (0 <= warmup < 1, 0 to disable) Default: 0.
        min_lr (float): The minimum learning rate. Default: 0.
        last_epoch (int): The index of last epoch. Default: -1.
        verbose (bool): Accepted and ignored. Default: ``False``.
    """

    def __init__(self, optimizer, inv_gamma=1., power=1., warmup=0., min_lr=0., last_epoch=-1, verbose=False):
        self.inv_gamma, self.power = inv_gamma, power
        _check_warmup(warmup)
        self.warmup, self.min_lr = warmup, min_lr
        super().__init__(optimizer, last_epoch)

    def _get_closed_form_lr(self):
        mult = (1 + self.last_epoch / self.inv_gamma) ** -self.power
        return [self._warmup() * max(self.min_lr, base_lr * mult) for base_lr in self.base_lrs]


class ExponentialLR(_ClosedFormLR):
    """Exponential decay by `decay` every num_steps steps, lr = base_lr (decay ** (1 / num_steps)) ** epoch floored at min_lr, times an
    exponential warmup (utils.py:196-234).

    Args:
        optimizer (Optimizer): Wrapped optimizer.
        num_steps (float): The number of steps to decay the learning rate by decay in.
        decay (float): The factor by which to decay the learning rate every num_steps steps. Default: 0.5.
        warmup (float): Exponential warmup factor (0 <= warmup < 1, 0 to disable) Default: 0.
        min_lr (float): The minimum learning rate. Default: 0.
        last_epoch (int): The index of last epoch. Default: -1.
        verbose (bool): Accepted and ignored. Default: ``False``.
    """

    def __init__(self, optimizer, num_steps, decay=0.5, warmup=0., min_lr=0., last_epoch=-1, verbose=False):
        self.num_steps, self.decay = num_steps, decay
        _check_warmup(warmup)
        self.warmup, self.min_lr = warmup, min_lr
        super().__init__(optimizer, last_epoch)

    def _get_closed_form_lr(self):
        mult = (self.decay ** (1 / self.num_steps)) ** self.last_epoch
        return [self._warmup() * max(self.min_lr, base_lr * mult) for base_lr in self.base_lrs]


class ConstantLRWithWarmup(_ClosedFormLR):
    """A constant learning rate times an exponential warmup 1 - warmup ** (epoch + 1) (utils.py:237-264).

    Args:
        optimizer (Optimizer): Wrapped optimizer.
        warmup (float): Exponential warmup factor (0 <= warmup < 1, 0 to disable) Default: 0.
        last_epoch (int): The index of last epoch. Default: -1.
        verbose (bool): Accepted and ignored. Default: ``False``.
    """

    def __init__(self, optimizer, warmup=0., last_epoch=-1, verbose=False):
        _check_warmup(warmup)
        self.warmup = warmup
        super().__init__(optimizer, last_epoch)

    def _get_closed_form_lr(self):
        return [self._warmup() * base_lr for base_lr in self.base_lrs]


def stratified_uniform(shape, group=0, groups=1, dtype=None, device=None):
    """Uniforms stratified along the last axis (utils.py:267-276): with n = shape[-1] * groups strata, element j of group `group` lies in
    stratum group + j * groups, i.e. (group + j * groups + u) / n."""
    if groups <= 0:
        raise ValueError(f"groups must be positive, got {groups}")
    if group < 0 or group >= groups:
        raise ValueError(f"group must be in [0, {groups})")
    n = shape[-1] * groups
    offsets = torch.arange(group, n, groups, dtype=dtype, device=device)
    return (offsets + torch.rand(shape, dtype=dtype, device=device)) / n


stratified_settings = threading.local()


@contextmanager
def enable_stratified(group=0, groups=1, disable=False):
    """Within the block, the sigma sample densities of this thread draw stratified uniforms of stratum group `group` of `groups`
    (utils.py:282-293); disable=True keeps plain uniforms."""
    try:
        stratified_settings.disable, stratified_settings.group, stratified_settings.groups = disable, group, groups
        yield
    finally:
        del stratified_settings.disable, stratified_settings.group, stratified_settings.groups


@contextmanager
def enable_stratified_accelerate(accelerator, disable=False):
    """enable_stratified with one stratum group per (process, gradient accumulation step) of a Hugging Face Accelerate `accelerator`
    (utils.py:296-310): group rank * acc_steps + step % acc_steps of world_size * acc_steps."""
    acc_steps = accelerator.gradient_state.num_steps
    group = accelerator.process_index * acc_steps + accelerator.step % acc_steps
    with enable_stratified(group, accelerator.num_processes * acc_steps, disable=disable):
        yield


def stratified_with_settings(shape, dtype=None, device=None):
    """torch.rand, or stratified_uniform under an enabled enable_stratified (utils.py:313-320)."""
    if getattr(stratified_settings, 'disable', True):
        return torch.rand(shape, dtype=dtype, device=device)
    return stratified_uniform(shape, stratified_settings.group, stratified_settings.groups, dtype=dtype, device=device)


# The sigma sample densities (utils.py:323-385).  Each is a few torch ops on `shape` values, issued in the reference's order and dtypes on
# the caller's device, so the same torch seed gives the reference's sigmas bit for bit on the same device.

def rand_log_normal(shape, loc=0., scale=1., device='cpu', dtype=torch.float32):
    """Lognormal samples: exp of the Normal(loc, scale) quantile of u * (1 - 2e-7) + 1e-7."""
    u = stratified_with_settings(shape, device=device, dtype=dtype) * (1 - 2e-7) + 1e-7
    return torch.distributions.Normal(loc, scale).icdf(u).exp()


def rand_log_logistic(shape, loc=0., scale=1., min_value=0., max_value=float('inf'), device='cpu', dtype=torch.float32):
    """Log-logistic samples truncated to [min_value, max_value], drawn in float64 by the inverse CDF, then cast to `dtype`."""
    lo = torch.as_tensor(min_value, device=device, dtype=torch.float64).log().sub(loc).div(scale).sigmoid()
    hi = torch.as_tensor(max_value, device=device, dtype=torch.float64).log().sub(loc).div(scale).sigmoid()
    u = stratified_with_settings(shape, device=device, dtype=torch.float64) * (hi - lo) + lo
    return u.logit().mul(scale).add(loc).exp().to(dtype)


def rand_log_uniform(shape, min_value, max_value, device='cpu', dtype=torch.float32):
    """Log-uniform samples on [min_value, max_value]."""
    lo, hi = math.log(min_value), math.log(max_value)
    return (stratified_with_settings(shape, device=device, dtype=dtype) * (hi - lo) + lo).exp()


def rand_v_diffusion(shape, sigma_data=1., min_value=0., max_value=float('inf'), device='cpu', dtype=torch.float32):
    """Samples of the v-diffusion (cosine) timestep distribution, truncated to [min_value, max_value]: sigma_data tan(u pi / 2)."""
    lo = math.atan(min_value / sigma_data) * 2 / math.pi
    hi = math.atan(max_value / sigma_data) * 2 / math.pi
    u = stratified_with_settings(shape, device=device, dtype=dtype) * (hi - lo) + lo
    return torch.tan(u * math.pi / 2) * sigma_data


def rand_cosine_interpolated(shape, image_d, noise_d_low, noise_d_high, sigma_data=1., min_value=1e-3, max_value=1e3, device='cpu',
                             dtype=torch.float32):
    """Samples of simple diffusion's interpolated cosine schedule: the logSNR of the cosine schedule shifted for noise_d_low and for
    noise_d_high at image size image_d, lerped by u, as sigma_data exp(-logsnr / 2)."""

    def cosine(t, logsnr_min, logsnr_max):
        t_min = math.atan(math.exp(-0.5 * logsnr_max))
        t_max = math.atan(math.exp(-0.5 * logsnr_min))
        return -2 * torch.log(torch.tan(t_min + t * (t_max - t_min)))

    def shifted(t, noise_d, logsnr_min, logsnr_max):
        shift = 2 * math.log(noise_d / image_d)
        return cosine(t, logsnr_min - shift, logsnr_max - shift) + shift

    logsnr_min = -2 * math.log(min_value / sigma_data)
    logsnr_max = -2 * math.log(max_value / sigma_data)
    u = stratified_with_settings(shape, device=device, dtype=dtype)
    logsnr = torch.lerp(shifted(u, noise_d_low, logsnr_min, logsnr_max), shifted(u, noise_d_high, logsnr_min, logsnr_max), u)
    return torch.exp(-logsnr / 2) * sigma_data


def rand_split_log_normal(shape, loc, scale_1, scale_2, device='cpu', dtype=torch.float32):
    """Split lognormal samples: exp(loc - scale_1 |n|) with probability scale_1 / (scale_1 + scale_2), else exp(loc + scale_2 |n|).
    Not stratified (the reference draws plain randn and rand here)."""
    n = torch.randn(shape, device=device, dtype=dtype).abs()
    u = torch.rand(shape, device=device, dtype=dtype)
    left = n * -scale_1 + loc
    right = n * scale_2 + loc
    return torch.where(u < scale_1 / (scale_1 + scale_2), left, right).exp()
