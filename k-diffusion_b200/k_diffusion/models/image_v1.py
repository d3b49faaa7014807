"""image_v1 U-Net denoiser -- parameter container + native forward, exact fp32 or with tf32 or fp16 convolutions and attention.

Constructor, forward signature and `state_dict()` layout follow the reference (k_diffusion/models/image_v1.py, layers.py:116-313),
so reference checkpoints load unchanged; the forward pass itself is executed by libkdb200.so (kdb_unet_*).  The torch modules
below only hold named parameters and buffers: none of their forward methods runs.  Inference only.  Precision: fp32 (the default,
every kernel exact fp32) or, by set_precision("tf32") or KDB200_PRECISION=tf32, every convolution and the d_head-64 attention on the tensor cores with tf32
operands and fp32 accumulation -- the arithmetic the reference's Conv2d gets on an H100 (cudnn.allow_tf32 defaults to True) -- or, by
set_precision("fp16") or KDB200_PRECISION=fp16, the same with fp16 operands (same significand width, narrower exponent range).
"""
import torch
from torch import nn

from .. import _native
from ..layers import FourierFeatures
from . import flags


def orthogonal_(module):
    nn.init.orthogonal_(module.weight)
    return module


class AdaGN(nn.Module):
    """layers.py:162-175"""

    def __init__(self, feats_in, c_out, num_groups, eps=1e-5, cond_key='cond'):
        super().__init__()
        self.num_groups, self.eps, self.cond_key = num_groups, eps, cond_key
        self.mapper = nn.Linear(feats_in, c_out * 2)
        nn.init.zeros_(self.mapper.weight)
        nn.init.zeros_(self.mapper.bias)


class ResConvBlock(nn.Module):
    """image_v1.py:15-29 (ConditionedResidualBlock, layers.py:151-159): main.{0..7} and skip"""

    def __init__(self, feats_in, c_in, c_mid, c_out, group_size=32, dropout_rate=0.):
        super().__init__()
        self.main = nn.Sequential(
            AdaGN(feats_in, c_in, max(1, c_in // group_size)), nn.GELU(), nn.Conv2d(c_in, c_mid, 3, padding=1), nn.Dropout2d(dropout_rate),
            AdaGN(feats_in, c_mid, max(1, c_mid // group_size)), nn.GELU(), nn.Conv2d(c_mid, c_out, 3, padding=1), nn.Dropout2d(dropout_rate))
        self.skip = nn.Identity() if c_in == c_out else orthogonal_(nn.Conv2d(c_in, c_out, 1, bias=False))
        nn.init.zeros_(self.main[-2].weight)
        nn.init.zeros_(self.main[-2].bias)


class SelfAttention2d(nn.Module):
    """layers.py:181-200"""

    def __init__(self, c_in, n_head, norm, dropout_rate=0.):
        super().__init__()
        assert c_in % n_head == 0
        self.norm_in = norm(c_in)
        self.n_head = n_head
        self.qkv_proj = nn.Conv2d(c_in, c_in * 3, 1)
        self.out_proj = nn.Conv2d(c_in, c_in, 1)
        self.dropout = nn.Dropout(dropout_rate)
        nn.init.zeros_(self.out_proj.weight)
        nn.init.zeros_(self.out_proj.bias)


class Downsample2d(nn.Module):
    """layers.py:251-257 ('linear' filter, reflect padding)"""

    def __init__(self):
        super().__init__()
        k1 = torch.tensor([[1 / 8, 3 / 8, 3 / 8, 1 / 8]])
        self.register_buffer('kernel', k1.T @ k1)


class Upsample2d(nn.Module):
    """layers.py:267-273"""

    def __init__(self):
        super().__init__()
        k1 = torch.tensor([[1 / 8, 3 / 8, 3 / 8, 1 / 8]]) * 2
        self.register_buffer('kernel', k1.T @ k1)


def _block(n_layers, feats_in, c_in, c_mid, c_out, self_attn, dropout_rate, group_size=32, head_size=64):
    mods = []
    for i in range(n_layers):
        my_c_in = c_in if i == 0 else c_mid
        my_c_out = c_mid if i < n_layers - 1 else c_out
        mods.append(ResConvBlock(feats_in, my_c_in, c_mid, my_c_out, group_size, dropout_rate))
        if self_attn:
            norm = lambda c, g=max(1, my_c_out // group_size): AdaGN(feats_in, c, g)
            mods.append(SelfAttention2d(my_c_out, max(1, my_c_out // head_size), norm, dropout_rate))
    return mods


def DBlock(n_layers, feats_in, c_in, c_mid, c_out, dropout_rate=0., downsample=False, self_attn=False):
    """image_v1.py:32-50: [Downsample2d | Identity, (ResConvBlock, [SelfAttention2d]) * n_layers]"""
    return nn.Sequential(Downsample2d() if downsample else nn.Identity(), *_block(n_layers, feats_in, c_in, c_mid, c_out, self_attn, dropout_rate))


def UBlock(n_layers, feats_in, c_in, c_mid, c_out, dropout_rate=0., upsample=False, self_attn=False):
    """image_v1.py:53-77: [(ResConvBlock, [SelfAttention2d]) * n_layers, Upsample2d | Identity]"""
    return nn.Sequential(*_block(n_layers, feats_in, c_in, c_mid, c_out, self_attn, dropout_rate), Upsample2d() if upsample else nn.Identity())


class UNet(nn.Module):
    """layers.py:298-303 (u_blocks innermost first)"""

    def __init__(self, d_blocks, u_blocks, skip_stages=0):
        super().__init__()
        self.d_blocks = nn.ModuleList(d_blocks)
        self.u_blocks = nn.ModuleList(u_blocks)
        self.skip_stages = skip_stages


class ImageDenoiserModelV1(_native.EngineCache, nn.Module):
    def __init__(self, c_in, feats_in, depths, channels, self_attn_depths, cross_attn_depths=None, mapping_cond_dim=0, unet_cond_dim=0,
                 cross_cond_dim=0, dropout_rate=0., patch_size=1, skip_stages=0, has_variance=False):
        super().__init__()
        if unet_cond_dim > 0 or cross_cond_dim > 0:
            raise NotImplementedError('unet_cond and cross-attention conditioning are not supported by the native image_v1 engine')
        self.c_in, self.channels, self.unet_cond_dim, self.patch_size, self.has_variance = c_in, channels, unet_cond_dim, patch_size, has_variance
        self.feats_in, self.depths, self.self_attn_depths, self.mapping_cond_dim = feats_in, list(depths), list(self_attn_depths), mapping_cond_dim
        self.dropout_rate = dropout_rate
        self.timestep_embed = FourierFeatures(1, feats_in)
        if mapping_cond_dim > 0:
            self.mapping_cond = nn.Linear(mapping_cond_dim, feats_in, bias=False)
        self.mapping = nn.Sequential(orthogonal_(nn.Linear(feats_in, feats_in)), nn.GELU(), orthogonal_(nn.Linear(feats_in, feats_in)), nn.GELU())
        self.proj_in = nn.Conv2d((c_in + unet_cond_dim) * patch_size ** 2, channels[max(0, skip_stages - 1)], 1)
        self.proj_out = nn.Conv2d(channels[max(0, skip_stages - 1)], c_in * patch_size ** 2 + (1 if has_variance else 0), 1)
        nn.init.zeros_(self.proj_out.weight)
        nn.init.zeros_(self.proj_out.bias)
        d_blocks, u_blocks = [], []
        for i in range(len(depths)):
            d_blocks.append(DBlock(depths[i], feats_in, channels[max(0, i - 1)], channels[i], channels[i], dropout_rate, i > skip_stages,
                                   self_attn_depths[i]))
        for i in range(len(depths)):
            my_c_in = channels[i] * 2 if i < len(depths) - 1 else channels[i]
            u_blocks.append(UBlock(depths[i], feats_in, my_c_in, channels[i], channels[max(0, i - 1)], dropout_rate, i > skip_stages,
                                   self_attn_depths[i]))
        self.u_net = UNet(d_blocks, reversed(u_blocks), skip_stages=skip_stages)
        self.precision = None
        self._engines = {}

    # ------------------------------------------------------------------ engine plumbing
    def engine_spec(self, augment):
        return dict(c_in=self.c_in, feats_in=self.feats_in, depths=self.depths, channels=self.channels, self_attn_depths=self.self_attn_depths,
                    mapping_cond_dim=self.mapping_cond_dim, augment=augment, patch_size=self.patch_size, skip_stages=self.u_net.skip_stages,
                    has_variance=self.has_variance)

    def engine(self, augment=False):
        """Native engine with the current parameters bound; `augment`: conditioning as KarrasAugmentWrapper forms it."""
        eng = self._engines.get(augment)
        if eng is None:
            eng = self._engines[augment] = _native.UNetEngine(self.engine_spec(augment))
        eng.bind(dict(self.state_dict(keep_vars=True)))
        return eng

    _PRECISIONS = {"fp32": "fp32", "float32": "fp32", "tf32": "tf32", "fp16": "fp16", "float16": "fp16"}

    def set_precision(self, precision):
        """'fp32' or None/'auto' (the exact fp32 path), 'tf32' or 'fp16' (tf32 / fp16 convolutions and attention); the U-Net has no bf16
        route."""
        if precision not in (None, "auto") and precision not in self._PRECISIONS:
            raise ValueError(f"the image_v1 U-Net runs at fp32, tf32 or fp16 (got precision {precision!r})")
        self.precision = None if precision in (None, "auto") else self._PRECISIONS[precision]
        return self

    def resolved_precision(self):
        p = flags.resolve_precision(self.precision, torch.float32)
        codes = {"fp32": _native.PREC_FP32, "tf32": _native.PREC_TF32, "fp16": _native.PREC_FP16}
        if p not in codes:
            raise ValueError(f"the image_v1 U-Net runs at fp32, tf32 or fp16 (resolved precision {p!r})")
        return codes[p]

    def param_groups(self, *args, **kwargs):
        raise NotImplementedError("training is out of scope for the H100 sampling path")

    def set_train_precision(self, precision):
        raise NotImplementedError("the image_v1 U-Net has no native training: only its forward is built")

    # ------------------------------------------------------------------ native front end
    def native_eval(self, x, sigma=None, aug_cond=None, class_cond=None, mapping_cond=None, precision=None, augment=False):
        """The native front end: validates one evaluation's inputs and returns its `_native.Evaluation` (the bound engine, `precision`
        or, when None, the resolved precision, and the engine's arguments).  `augment`: the evaluation KarrasAugmentWrapper asks for,
        whose engine forms mapping_cond = cat([aug_cond or zeros(B, 9), mapping_cond]) in its conditioning kernel."""
        _native.check_input(x, sigma, self.training and self.dropout_rate > 0)
        if torch.is_grad_enabled() and x.requires_grad:
            _native.unet_has_no_derivative()
        if aug_cond is not None and not augment:
            raise TypeError("aug_cond needs the KarrasAugmentWrapper")
        if class_cond is not None:
            raise TypeError("the image_v1 U-Net takes no class_cond")
        user_mapping_cond_dim = self.mapping_cond_dim - (9 if augment else 0)
        if mapping_cond is not None and user_mapping_cond_dim <= 0:
            raise ValueError("this model takes no mapping_cond")
        _native.require_cond(None, mapping_cond, False, augment and user_mapping_cond_dim > 0)
        return _native.Evaluation(self.engine(augment), self.resolved_precision() if precision is None else precision, x, sigma, aug_cond,
                                  None, mapping_cond, False, True)

    def denoise(self, x, sigma, sigma_data, mapping_cond=None, out=None):
        """Fused Karras-preconditioned evaluation c_skip x + c_out F(c_in x, sigma) (layers.py:88-90)."""
        return self.native_eval(x, sigma, mapping_cond=mapping_cond).forward(float(sigma_data), out)

    denoise_jvp = denoise_vjp = _native.unet_has_no_derivative

    def forward(self, input, sigma, mapping_cond=None, unet_cond=None, cross_cond=None, cross_cond_padding=None, return_variance=False):
        """reference image_v1.py:135-157"""
        if unet_cond is not None or cross_cond is not None:
            raise NotImplementedError('unet_cond and cross-attention conditioning are not supported by the native image_v1 engine')
        if return_variance:
            raise NotImplementedError('the variance output is a training quantity; the native engine returns the denoised channels only')
        return self.native_eval(input, sigma, mapping_cond=mapping_cond).forward(0.0)
