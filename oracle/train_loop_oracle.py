"""The reference's sigma sample densities (utils.py:267-385, config.py:234-268) restated as plain functions of a config: the torch op
sequence, dtypes and draw order of the reference, with stratification passed as an argument instead of thread-local state.
oracle/make_golden_train_loop.py pins this restatement to the reference on the CPU; on the GPU the product is held to it bit for bit."""
import math

import torch


def _uniform(shape, strat, dtype, device):
    """strat None: torch.rand; (group, groups): the stratified uniform of that group"""
    if strat is None:
        return torch.rand(shape, dtype=dtype, device=device)
    group, groups = strat
    n = shape[-1] * groups
    return (torch.arange(group, n, groups, dtype=dtype, device=device) + torch.rand(shape, dtype=dtype, device=device)) / n


def _pick(d, new, old):
    return d[new] if new in d else d[old]


def sample_density(config, shape, device, strat=None, dtype=torch.float32):
    """Training sigmas of `shape` from config['sigma_sample_density'] of a model config."""
    sd, sigma_data = config['sigma_sample_density'], config['sigma_data']
    kind = sd['type']
    if kind == 'lognormal':
        u = _uniform(shape, strat, dtype, device) * (1 - 2e-7) + 1e-7
        return torch.distributions.Normal(_pick(sd, 'mean', 'loc'), _pick(sd, 'std', 'scale')).icdf(u).exp()
    if kind == 'loglogistic':
        loc = sd['loc'] if 'loc' in sd else math.log(sigma_data)
        scale = sd.get('scale', 0.5)
        cdf = [torch.as_tensor(sd.get(k, v), device=device, dtype=torch.float64).log().sub(loc).div(scale).sigmoid()
               for k, v in (('min_value', 0.), ('max_value', float('inf')))]
        u = _uniform(shape, strat, torch.float64, device) * (cdf[1] - cdf[0]) + cdf[0]
        return u.logit().mul(scale).add(loc).exp().to(dtype)
    if kind == 'loguniform':
        lo = math.log(sd['min_value'] if 'min_value' in sd else config['sigma_min'])
        hi = math.log(sd['max_value'] if 'max_value' in sd else config['sigma_max'])
        return (_uniform(shape, strat, dtype, device) * (hi - lo) + lo).exp()
    if kind in ('v-diffusion', 'cosine'):
        lo = math.atan(sd.get('min_value', 1e-3) / sigma_data) * 2 / math.pi
        hi = math.atan(sd.get('max_value', 1e3) / sigma_data) * 2 / math.pi
        u = _uniform(shape, strat, dtype, device) * (hi - lo) + lo
        return torch.tan(u * math.pi / 2) * sigma_data
    if kind == 'split-lognormal':
        loc, s1, s2 = _pick(sd, 'mean', 'loc'), _pick(sd, 'std_1', 'scale_1'), _pick(sd, 'std_2', 'scale_2')
        n = torch.randn(shape, device=device, dtype=dtype).abs()
        u = torch.rand(shape, device=device, dtype=dtype)
        return torch.where(u < s1 / (s1 + s2), n * -s1 + loc, n * s2 + loc).exp()
    if kind == 'cosine-interpolated':
        size = max(config['input_size'])
        lo, hi = sd.get('min_value', min(config['sigma_min'], 1e-3)), sd.get('max_value', max(config['sigma_max'], 1e3))
        image_d = sd.get('image_d', size)
        logsnr_min, logsnr_max = -2 * math.log(lo / sigma_data), -2 * math.log(hi / sigma_data)
        u = _uniform(shape, strat, dtype, device)

        def logsnr(noise_d):
            shift = 2 * math.log(noise_d / image_d)
            t0, t1 = math.atan(math.exp(-0.5 * (logsnr_max - shift))), math.atan(math.exp(-0.5 * (logsnr_min - shift)))
            return -2 * torch.log(torch.tan(t0 + u * (t1 - t0))) + shift

        return torch.exp(-torch.lerp(logsnr(sd.get('noise_d_low', 32)), logsnr(sd.get('noise_d_high', size)), u) / 2) * sigma_data
    raise ValueError('Unknown sample density type')
