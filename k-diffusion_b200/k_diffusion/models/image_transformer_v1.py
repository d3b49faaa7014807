"""image_transformer_v1 denoiser -- parameter container + native forward.

Constructor signature, `forward` signature and `state_dict()` layout follow the reference
(k_diffusion/models/image_transformer_v1.py:280-344) so reference checkpoints load unchanged.  The forward runs on the
image_transformer_v2 engine (libkdb200.so, KdbModelConfig.family = image_transformer_v1): v1 is a one-level v2 model with global
attention, a mapping network of depth 2 and width d_model, whose QKNorm and interleaved AxialRoPE become the engine's cosine-sim
attention and half-split RoPE through tables kdb_model_finalize derives from v1's own weights.  Inference only.

Deviations from the reference, each refused with an error instead of computed:
  * d_ff = 0 (the reference's config placeholder, which load_config replaces): the feed-forward blocks would be identities;
  * d_model not a multiple of 64 (the reference's d_head is 64; a partial head is not an attention head);
  * mapping_cond: v1's forward takes none, so the augment wrapper (which passes one) is refused by config.load_config.
`qk_norm.scale` is never clamped in place (the reference's proj_() does so on every forward): the engine applies min(scale, ln 100)
in its derived scale table, and writing the parameter would invalidate the bound engine on every call.
"""
import math

import torch
from torch import nn

from .. import _native
from .image_transformer_v2 import GlobalAttentionSpec, LevelSpec, MappingSpec, TransformerEngineModel, _Buffer, _Node, _linear

D_HEAD = 64


def _freqs_pixel_log(n_heads, dim, max_freq=10.0):
    # axial_rope.py:77-82: log frequencies linspace(ln pi, ln(max_freq pi / 2)) per head, shape [n_heads, dim // 4]
    return torch.linspace(math.log(math.pi), math.log(max_freq * math.pi / 2), dim // 4).expand(n_heads, dim // 4).clone()


def _block(d_model, d_ff):
    n_heads = d_model // D_HEAD
    return _Node(
        self_attn=_Node(
            norm=_Node(linear=_linear(d_model, d_model, zero=True)),
            qkv_proj=_linear(d_model * 3, d_model),
            qk_norm=_Node(scale=torch.full((n_heads,), math.log(10.0))),
            pos_emb=_Node(freqs_h=_freqs_pixel_log(n_heads, D_HEAD), freqs_w=_freqs_pixel_log(n_heads, D_HEAD)),
            out_proj=_linear(d_model, d_model, zero=True),
        ),
        ff=_Node(
            norm=_Node(linear=_linear(d_model, d_model, zero=True)),
            up_proj=_linear(d_ff * 2, d_model),
            down_proj=_linear(d_model, d_ff, zero=True),
        ),
    )


class ImageTransformerDenoiserModelV1(TransformerEngineModel):
    family = _native.FAMILY_ITV1
    kind = "image_transformer_v1"
    dtype_key = "in_proj.weight"

    def __init__(self, n_layers, d_model, d_ff, in_features, out_features, patch_size, num_classes=0, dropout=0.0, sigma_data=1.0):
        super().__init__()
        if d_model % D_HEAD != 0:
            raise ValueError(f"image_transformer_v1: width {d_model} is not a multiple of d_head {D_HEAD}")
        if d_ff <= 0:
            raise ValueError(f"image_transformer_v1: d_ff = {d_ff} gives identity feed-forward blocks; not supported by the native engine")
        patch_size = tuple(patch_size) if not isinstance(patch_size, int) else (patch_size, patch_size)
        self.sigma_data = sigma_data
        self.num_classes = num_classes
        self.levels = [LevelSpec(n_layers, d_model, d_ff, GlobalAttentionSpec(D_HEAD), dropout)]
        self.mapping_spec = MappingSpec(2, d_model, d_ff, dropout)        # MappingNetwork(2, d_model, d_ff) (:293)
        self.in_channels, self.out_channels, self.patch_size, self.mapping_cond_dim = in_features, out_features, patch_size, 0
        n_patch = patch_size[0] * patch_size[1]

        self.time_emb = _Node(weight=_Buffer(torch.randn(d_model // 2, 1)))       # layers.FourierFeatures(1, d_model)
        self.time_in_proj = _linear(d_model, d_model)
        self.aug_emb = _Node(weight=_Buffer(torch.randn(d_model // 2, 9)))        # layers.FourierFeatures(9, d_model)
        self.aug_in_proj = _linear(d_model, d_model)
        self.class_emb = _Node(weight=torch.randn(num_classes, d_model)) if num_classes else None
        self.mapping_cond_in_proj = None
        self.mapping = _Node(
            in_norm=_Node(scale=torch.ones(d_model)),
            blocks=nn.ModuleList([
                _Node(norm=_Node(scale=torch.ones(d_model)), up_proj=_linear(d_ff * 2, d_model), down_proj=_linear(d_model, d_ff, zero=True))
                for _ in range(2)]),
            out_norm=_Node(scale=torch.ones(d_model)),
        )
        self.in_proj = _linear(d_model, in_features * n_patch)                    # input features in Patching's (c i j) order
        self.blocks = nn.ModuleList([_block(d_model, d_ff) for _ in range(n_layers)])
        self.out_norm = _Node(scale=torch.ones(d_model))
        self.out_proj = _linear(out_features * n_patch, d_model, zero=True)       # output features in Unpatching's (c i j) order

        self.precision = None        # None -> flags.resolve_precision ("auto" unless KDB200_PRECISION is set)
        self._engines = {}

    def param_groups(self, *args, **kwargs):
        """Training image_transformer_v1 is not built (its parameters carry none of the reference's weight-decay / mapping tags)."""
        raise NotImplementedError("image_transformer_v1: training is not built; parameter gradients exist for image_transformer_v2 only")

    def _check_cond(self, class_cond, mapping_cond):
        if mapping_cond is not None:
            raise TypeError("image_transformer_v1 takes no mapping_cond (reference forward(x, sigma, aug_cond=None, class_cond=None))")
        super()._check_cond(class_cond, mapping_cond)

    def forward(self, x, sigma, aug_cond=None, class_cond=None):
        """F(x, sigma): the raw inner model (reference :317-344)."""
        return self._run(x, sigma, 0.0, aug_cond, class_cond, None)
