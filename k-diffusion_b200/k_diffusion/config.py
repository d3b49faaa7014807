"""Config loading / model factory for the path in scope (reference: k_diffusion/config.py:23-231).

make_sample_density (config.py:234-268) builds the sigma sample density of train.py's step.
Accepts the reference's JSON files, dicts, and `.safetensors` checkpoints carrying the config in
their metadata.  `image_transformer_v2`, `image_transformer_v1` and `image_v1` can be built.
"""
import json
import math
from functools import partial
from pathlib import Path

from . import augmentation, layers, models, utils

_V2_MODEL_DEFAULTS = dict(mapping_width=256, mapping_depth=2, mapping_d_ff=None, mapping_cond_dim=0, mapping_dropout_rate=0.,
                          d_ffs=None, self_attns=None, dropout_rate=None, augment_wrapper=False, skip_stages=0, has_variance=False)
_V1_MODEL_DEFAULTS = dict(patch_size=1, augment_wrapper=True, mapping_cond_dim=0, unet_cond_dim=0, cross_cond_dim=0, cross_attn_depths=None,
                          skip_stages=0, has_variance=False)
_V1_OPT_DEFAULTS = dict(type='adamw', lr=1e-4, betas=[0.95, 0.999], eps=1e-6, weight_decay=1e-3)
# keys make_model needs that have no default: the reference fails on them later, in make_model (KeyError)
_V1_REQUIRED = ('input_channels', 'input_size', 'mapping_out', 'depths', 'channels', 'self_attn_depths')
_V2_OPT_DEFAULTS = dict(type='adamw', lr=5e-4, betas=[0.9, 0.99], eps=1e-8, weight_decay=1e-4)
_ITV1_MODEL_DEFAULTS = dict(d_ff=0, augment_wrapper=False, skip_stages=0, has_variance=False)
_COMMON_DEFAULTS = {
    'model': dict(sigma_data=1., dropout_rate=0., augment_prob=0., loss_config='karras', loss_weighting='karras', loss_scales=1),
    'dataset': dict(type='imagefolder', num_classes=0, cond_dropout_rate=0.1),
    'optimizer': dict(type='adamw', lr=1e-4, betas=[0.9, 0.999], eps=1e-8, weight_decay=1e-4),
    'lr_sched': dict(type='constant', warmup=0.),
    'ema_sched': dict(type='inverse', power=0.6667, max_value=0.9999),
}


def _overlay(base, head):
    """Recursive dict merge, `head` wins; non-dict values (lists included) are replaced (jsonmerge default)."""
    if not (isinstance(base, dict) and isinstance(head, dict)):
        return head
    out = dict(base)
    for k, v in head.items():
        out[k] = _overlay(base[k], v) if k in base else v
    return out


def round_to_power_of_two(x, tol):
    """The nearest multiple of 2**k to x for the largest k < ceil(log2 x) that lands within relative `tol` of x; x rounded to an integer
    when none does (the d_ff default of image_transformer_v1 configs, reference config.py:11-20)."""
    for k in range(math.ceil(math.log2(x)) - 1, -1, -1):
        step = 2 ** k
        candidate = round(x / step) * step
        if abs(candidate - x) <= tol * abs(x):
            return candidate
    return round(x)


def _read(path_or_dict):
    if isinstance(path_or_dict, dict):
        return path_or_dict
    file = Path(path_or_dict)
    if file.suffix == '.safetensors':
        from safetensors import safe_open
        with safe_open(str(file), framework='pt') as f:
            return json.loads(f.metadata()['config'])
    return json.loads(file.read_text())


def load_config(path_or_dict):
    config = _read(path_or_dict)
    kind = config['model']['type']
    if kind == 'image_v1':
        missing = [k for k in _V1_REQUIRED if k not in config['model']]
        if missing:
            raise ValueError(f'image_v1 config lacks {missing} (make_model needs them and they have no default)')
        return _overlay(_COMMON_DEFAULTS, _overlay({'model': _V1_MODEL_DEFAULTS, 'optimizer': _V1_OPT_DEFAULTS}, config))
    if kind == 'image_transformer_v1':
        config = _overlay({'model': _ITV1_MODEL_DEFAULTS, 'optimizer': _V2_OPT_DEFAULTS}, config)
        m = config['model']
        if m['augment_wrapper']:
            raise ValueError('image_transformer_v1 with augment_wrapper: the wrapper passes mapping_cond, which the v1 model does not take')
        if m['width'] % 64 != 0:
            raise ValueError(f"image_transformer_v1 width {m['width']} is not a multiple of its d_head 64")
        if not m['d_ff']:
            m['d_ff'] = round_to_power_of_two(m['width'] * 8 / 3, tol=0.05)
        return _overlay(_COMMON_DEFAULTS, config)
    if kind != 'image_transformer_v2':
        raise ValueError(f'model type {kind!r} is out of scope for the H100 sampling path (image_transformer_v2, image_transformer_v1 and '
                         'image_v1 only)')
    config = _overlay({'model': _V2_MODEL_DEFAULTS, 'optimizer': _V2_OPT_DEFAULTS}, config)
    m = config['model']
    n = len(m['widths'])
    if not m['mapping_d_ff']:
        m['mapping_d_ff'] = m['mapping_width'] * 3
    if not m['d_ffs']:
        m['d_ffs'] = [w * 3 for w in m['widths']]
    if not m['self_attns']:
        m['self_attns'] = [{"type": "neighborhood", "d_head": 64, "kernel_size": 7}] * (n - 1) + [{"type": "global", "d_head": 64}]
    if m['dropout_rate'] is None:
        m['dropout_rate'] = [0.0] * n
    elif isinstance(m['dropout_rate'], float):
        m['dropout_rate'] = [m['dropout_rate']] * n
    return _overlay(_COMMON_DEFAULTS, config)


def _attn_spec(a):
    v2 = models.image_transformer_v2
    if a['type'] == 'global':
        return v2.GlobalAttentionSpec(a.get('d_head', 64))
    if a['type'] == 'neighborhood':
        return v2.NeighborhoodAttentionSpec(a.get('d_head', 64), a.get('kernel_size', 7))
    if a['type'] == 'shifted-window':
        return v2.ShiftedWindowAttentionSpec(a.get('d_head', 64), a['window_size'])
    if a['type'] == 'none':
        return v2.NoAttentionSpec()
    raise ValueError(f'unsupported self attention type {a["type"]}')


def make_model(config):
    num_classes = config['dataset']['num_classes']
    m = config['model']
    if m['type'] == 'image_v1':
        if m['unet_cond_dim'] > 0 or m['cross_cond_dim'] > 0:
            raise NotImplementedError('unet_cond_dim / cross_cond_dim > 0: the native image_v1 engine has no U-Net or cross-attention conditioning')
        model = models.ImageDenoiserModelV1(
            m['input_channels'], m['mapping_out'], m['depths'], m['channels'], m['self_attn_depths'], m['cross_attn_depths'],
            patch_size=m['patch_size'], dropout_rate=m['dropout_rate'], mapping_cond_dim=m['mapping_cond_dim'] + (9 if m['augment_wrapper'] else 0),
            unet_cond_dim=m['unet_cond_dim'], cross_cond_dim=m['cross_cond_dim'], skip_stages=m['skip_stages'], has_variance=m['has_variance'])
        return augmentation.KarrasAugmentWrapper(model) if m['augment_wrapper'] else model
    if m['type'] == 'image_transformer_v1':
        if m.get('augment_wrapper'):
            raise ValueError('image_transformer_v1 with augment_wrapper: the wrapper passes mapping_cond, which the v1 model does not take')
        return models.ImageTransformerDenoiserModelV1(
            n_layers=m['depth'], d_model=m['width'], d_ff=m['d_ff'], in_features=m['input_channels'], out_features=m['input_channels'],
            patch_size=m['patch_size'], num_classes=num_classes + 1 if num_classes else 0, dropout=m['dropout_rate'],
            sigma_data=m['sigma_data'])
    if m['type'] != 'image_transformer_v2':
        raise ValueError(f'unsupported model type {m["type"]}')
    v2 = models.image_transformer_v2
    per_level = (m['depths'], m['widths'], m['d_ffs'], m['self_attns'], m['dropout_rate'])
    assert all(len(p) == len(m['widths']) for p in per_level)
    levels = [v2.LevelSpec(d, w, f, _attn_spec(a), p) for d, w, f, a, p in zip(*per_level)]
    mapping = v2.MappingSpec(m['mapping_depth'], m['mapping_width'], m['mapping_d_ff'], m['mapping_dropout_rate'])
    return models.ImageTransformerDenoiserModelV2(
        levels=levels, mapping=mapping, in_channels=m['input_channels'], out_channels=m['input_channels'],
        patch_size=m['patch_size'], num_classes=num_classes + 1 if num_classes else 0, mapping_cond_dim=m['mapping_cond_dim'])


def make_denoiser_wrapper(config):
    """reference config.py:216-232; the three wrappers differ in their training loss only, `forward` (what sampling calls) is shared"""
    m = config['model']
    sigma_data, has_variance, loss_config = m.get('sigma_data', 1.), m.get('has_variance', False), m.get('loss_config', 'karras')
    if loss_config == 'karras':
        weighting = m.get('loss_weighting', 'karras')
        if not has_variance:
            return partial(layers.Denoiser, sigma_data=sigma_data, weighting=weighting, scales=m.get('loss_scales', 1))
        return partial(layers.DenoiserWithVariance, sigma_data=sigma_data, weighting=weighting)
    if loss_config == 'simple':
        if has_variance:
            raise ValueError('Simple loss config does not support a variance output')
        return partial(layers.SimpleLossDenoiser, sigma_data=sigma_data)
    raise ValueError('Unknown loss config type')


def _first(d, *keys):
    """d[key] of the first of `keys` present; a KeyError naming the last when none is (the reference's 'mean' if 'mean' in d else d['loc'])."""
    for k in keys[:-1]:
        if k in d:
            return d[k]
    return d[keys[-1]]


def make_sample_density(config):
    """The sigma sample density of a model config (config['model'] of a loaded config; config.py:234-268): a function of (shape, device=,
    dtype=) drawing training sigmas, one of utils.rand_* with the config's parameters bound.  `sigma_sample_density.type`: lognormal
    (mean | loc, std | scale), loglogistic (loc = log sigma_data, scale = 0.5, min_value = 0, max_value = inf), loguniform (min_value |
    sigma_min, max_value | sigma_max), v-diffusion or cosine (min_value = 1e-3, max_value = 1e3), split-lognormal (mean | loc, std_1 | scale_1,
    std_2 | scale_2) or cosine-interpolated (min_value = min(sigma_min, 1e-3), max_value = max(sigma_max, 1e3), image_d = max(input_size),
    noise_d_low = 32, noise_d_high = max(input_size)); any other type raises ValueError."""
    sd = config['sigma_sample_density']
    sigma_data = config['sigma_data']
    kind = sd['type']
    if kind == 'lognormal':
        return partial(utils.rand_log_normal, loc=_first(sd, 'mean', 'loc'), scale=_first(sd, 'std', 'scale'))
    if kind == 'loglogistic':
        return partial(utils.rand_log_logistic, loc=sd['loc'] if 'loc' in sd else math.log(sigma_data), scale=sd.get('scale', 0.5), min_value=sd.get('min_value', 0.), max_value=sd.get('max_value', float('inf')))
    if kind == 'loguniform':
        return partial(utils.rand_log_uniform, min_value=sd['min_value'] if 'min_value' in sd else config['sigma_min'], max_value=sd['max_value'] if 'max_value' in sd else config['sigma_max'])
    if kind in {'v-diffusion', 'cosine'}:
        return partial(utils.rand_v_diffusion, sigma_data=sigma_data, min_value=sd.get('min_value', 1e-3), max_value=sd.get('max_value', 1e3))
    if kind == 'split-lognormal':
        return partial(utils.rand_split_log_normal, loc=_first(sd, 'mean', 'loc'), scale_1=_first(sd, 'std_1', 'scale_1'),
                       scale_2=_first(sd, 'std_2', 'scale_2'))
    if kind == 'cosine-interpolated':
        size = max(config['input_size'])
        return partial(utils.rand_cosine_interpolated, image_d=sd.get('image_d', size), noise_d_low=sd.get('noise_d_low', 32),
                       noise_d_high=sd.get('noise_d_high', size), sigma_data=sigma_data,
                       min_value=sd.get('min_value', min(config['sigma_min'], 1e-3)), max_value=sd.get('max_value', max(config['sigma_max'], 1e3)))
    raise ValueError('Unknown sample density type')
