"""Config loading / model factory for the path in scope (reference: k_diffusion/config.py:23-231).

Accepts the reference's JSON files, dicts, and `.safetensors` checkpoints carrying the config in
their metadata.  Only `image_transformer_v2` can be built; the other model families are out of scope.
"""
import json
from functools import partial
from pathlib import Path

from . import layers, models

_V2_MODEL_DEFAULTS = dict(mapping_width=256, mapping_depth=2, mapping_d_ff=None, mapping_cond_dim=0, mapping_dropout_rate=0.,
                          d_ffs=None, self_attns=None, dropout_rate=None, augment_wrapper=False, skip_stages=0, has_variance=False)
_V2_OPT_DEFAULTS = dict(type='adamw', lr=5e-4, betas=[0.9, 0.99], eps=1e-8, weight_decay=1e-4)
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
    if kind != 'image_transformer_v2':
        raise ValueError(f'model type {kind!r} is out of scope for the H100 sampling path (only image_transformer_v2)')
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
