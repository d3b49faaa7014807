"""image_transformer_v2 (HDiT) denoiser -- parameter container + native forward.

Constructor signature, spec dataclasses and `state_dict()` layout follow the reference
(k_diffusion/models/image_transformer_v2.py:626-706) so reference checkpoints load unchanged; the
forward pass itself (:721-762) is executed by libkdb200.so.  This module holds no layer logic: it
is a tree of named parameters whose names reproduce the reference keys.  Inference only.
"""
import math
from dataclasses import dataclass
from typing import Union

import torch
from torch import nn

from .. import _native
from . import flags


@dataclass
class GlobalAttentionSpec:
    d_head: int


@dataclass
class NeighborhoodAttentionSpec:
    d_head: int
    kernel_size: int


@dataclass
class ShiftedWindowAttentionSpec:
    d_head: int
    window_size: int


@dataclass
class NoAttentionSpec:
    pass


@dataclass
class LevelSpec:
    depth: int
    width: int
    d_ff: int
    self_attn: Union[GlobalAttentionSpec, NeighborhoodAttentionSpec, ShiftedWindowAttentionSpec, NoAttentionSpec]
    dropout: float


@dataclass
class MappingSpec:
    depth: int
    width: int
    d_ff: int
    dropout: float


class _Node(nn.Module):
    """A bag of named parameters / buffers / children; exists only to shape state_dict keys."""

    def __init__(self, **items):
        super().__init__()
        for name, value in items.items():
            if isinstance(value, nn.Module):
                self.add_module(name, value)
            elif isinstance(value, _Buffer):
                self.register_buffer(name, value.tensor)
            else:
                self.register_parameter(name, nn.Parameter(value))


class _Buffer:
    def __init__(self, tensor):
        self.tensor = tensor


def _linear(n_out, n_in, zero=False):
    """nn.Linear(bias=False) weight: U(-1/sqrt(in), 1/sqrt(in)), or zeros where the reference zero-inits."""
    w = torch.zeros(n_out, n_in)
    if not zero:
        bound = 1.0 / math.sqrt(n_in)
        w.uniform_(-bound, bound)
    return _Node(weight=w)


def _rope_freqs(d_head, n_heads):
    # AxialRoPE(d_head // 2, n_heads): log-spaced pi .. 10 pi, interleaved over heads (reference :234-240)
    n = n_heads * (d_head // 2) // 4
    f = torch.linspace(math.log(math.pi), math.log(10.0 * math.pi), n + 1)[:-1].exp()
    return f.view(-1, n_heads).T.contiguous()


def _attn_kind(spec):
    if isinstance(spec, GlobalAttentionSpec):
        return "global", 0
    if isinstance(spec, NeighborhoodAttentionSpec):
        return "neighborhood", spec.kernel_size
    if isinstance(spec, ShiftedWindowAttentionSpec):
        return "shifted-window", spec.window_size
    if isinstance(spec, NoAttentionSpec):
        return "none", 0
    raise ValueError(f"unsupported self attention spec {spec}")


def _layer(spec, cond_width):
    kind, _ = _attn_kind(spec.self_attn)
    parts = {}
    if kind != "none":
        d_head = spec.self_attn.d_head
        n_heads = spec.width // d_head
        parts["self_attn"] = _Node(
            norm=_Node(linear=_linear(spec.width, cond_width, zero=True)),
            qkv_proj=_linear(spec.width * 3, spec.width),
            scale=torch.full([n_heads], 10.0),
            pos_emb=_Node(freqs=_Buffer(_rope_freqs(d_head, n_heads))),
            out_proj=_linear(spec.width, spec.width, zero=True),
        )
    parts["ff"] = _Node(
        norm=_Node(linear=_linear(spec.width, cond_width, zero=True)),
        up_proj=_linear(spec.d_ff * 2, spec.width),
        down_proj=_linear(spec.width, spec.d_ff, zero=True),
    )
    return _Node(**parts)


def _level(spec, cond_width):
    return nn.ModuleList([_layer(spec, cond_width) for _ in range(spec.depth)])


class ImageTransformerDenoiserModelV2(nn.Module):
    def __init__(self, levels, mapping, in_channels, out_channels, patch_size, num_classes=0, mapping_cond_dim=0):
        super().__init__()
        levels = list(levels)
        patch_size = tuple(patch_size) if not isinstance(patch_size, int) else (patch_size, patch_size)
        self.num_classes = num_classes
        self.levels, self.mapping_spec = levels, mapping
        self.in_channels, self.out_channels, self.patch_size, self.mapping_cond_dim = in_channels, out_channels, patch_size, mapping_cond_dim
        for spec in levels:
            _attn_kind(spec.self_attn)           # raises ValueError on unsupported specs, like the reference (:693)
        mw = mapping.width
        w0 = levels[0].width
        n_patch = patch_size[0] * patch_size[1]

        self.patch_in = _Node(proj=_linear(w0, in_channels * n_patch))
        self.time_emb = _Node(weight=_Buffer(torch.randn(mw // 2, 1)))            # layers.FourierFeatures(1, mw)
        self.time_in_proj = _linear(mw, mw)
        self.aug_emb = _Node(weight=_Buffer(torch.randn(mw // 2, 9)))             # layers.FourierFeatures(9, mw)
        self.aug_in_proj = _linear(mw, mw)
        self.class_emb = _Node(weight=torch.randn(num_classes, mw)) if num_classes else None
        self.mapping_cond_in_proj = _linear(mw, mapping_cond_dim) if mapping_cond_dim else None
        self.mapping = _Node(
            in_norm=_Node(scale=torch.ones(mw)),
            blocks=nn.ModuleList([
                _Node(norm=_Node(scale=torch.ones(mw)), up_proj=_linear(mapping.d_ff * 2, mw), down_proj=_linear(mw, mapping.d_ff, zero=True))
                for _ in range(mapping.depth)]),
            out_norm=_Node(scale=torch.ones(mw)),
        )
        self.down_levels = nn.ModuleList([_level(s, mw) for s in levels[:-1]])
        self.up_levels = nn.ModuleList([_level(s, mw) for s in levels[:-1]])
        self.mid_level = _level(levels[-1], mw)
        self.merges = nn.ModuleList([_Node(proj=_linear(b.width, a.width * 4)) for a, b in zip(levels[:-1], levels[1:])])
        self.splits = nn.ModuleList([_Node(proj=_linear(a.width * 4, b.width), fac=torch.ones(1) * 0.5) for a, b in zip(levels[:-1], levels[1:])])
        self.out_norm = _Node(scale=torch.ones(w0))
        self.patch_out = _Node(proj=_linear(out_channels * n_patch, w0, zero=True))

        self.precision = None        # None -> flags.resolve_precision ("auto" unless KDB200_PRECISION is set)
        self._engine_obj = None

    # ------------------------------------------------------------------ engine plumbing
    def __getstate__(self):
        state = self.__dict__.copy()
        state["_engine_obj"] = None
        return state

    def __deepcopy__(self, memo):
        import copy
        eng, self._engine_obj = self._engine_obj, None
        try:
            cls = self.__class__
            new = cls.__new__(cls)
            memo[id(self)] = new
            new.__dict__ = copy.deepcopy(self.__dict__, memo)
        finally:
            self._engine_obj = eng
        return new

    def engine_spec(self):
        lv = []
        for s in self.levels:
            kind, param = _attn_kind(s.self_attn)
            lv.append(dict(width=s.width, depth=s.depth, d_ff=s.d_ff, attn=kind, d_head=getattr(s.self_attn, "d_head", 0), attn_param=param))
        return dict(levels=lv, in_channels=self.in_channels, out_channels=self.out_channels, patch_size=self.patch_size,
                    mapping_width=self.mapping_spec.width, mapping_depth=self.mapping_spec.depth, mapping_d_ff=self.mapping_spec.d_ff,
                    num_classes=self.num_classes, mapping_cond_dim=self.mapping_cond_dim)

    def engine(self):
        """Native engine with the current parameters bound (rebinds only after the parameters changed)."""
        if self._engine_obj is None:
            self._engine_obj = _native.Engine(self.engine_spec())
        tensors = dict(self.state_dict(keep_vars=True))
        self._engine_obj.bind(tensors)
        return self._engine_obj

    def set_precision(self, precision):
        """'fp32' (exact path, parity gate), 'bf16' (tensor-core path) or None/'auto'."""
        self.precision = None if precision in (None, "auto") else precision
        return self

    def resolved_precision(self):
        p = flags.resolve_precision(self.precision, self.patch_in.proj.weight.dtype)
        return _native.PREC_BF16 if p == "bf16" else _native.PREC_FP32

    def param_groups(self, *args, **kwargs):
        raise NotImplementedError("training is out of scope for the H100 sampling path")

    # ------------------------------------------------------------------ forward
    def _check_cond(self, class_cond, mapping_cond):
        if class_cond is None and self.class_emb is not None:
            raise ValueError("class_cond must be specified if num_classes > 0")
        if mapping_cond is None and self.mapping_cond_in_proj is not None:
            raise ValueError("mapping_cond must be specified if mapping_cond_dim > 0")

    def conditioning(self, sigma, aug_cond=None, class_cond=None, mapping_cond=None):
        """Conditioning table rows for `sigma` [rows] (mapping network + all AdaRMSNorm scales)."""
        self._check_cond(class_cond, mapping_cond)
        return self.engine().conditioning(sigma, aug_cond, class_cond if self.class_emb is not None else None,
                                          mapping_cond if self.mapping_cond_in_proj is not None else None)

    def _run(self, x, sigma, sigma_data, aug_cond, class_cond, mapping_cond, out=None):
        _native.require_cuda(x, sigma)
        if x.ndim != 4:
            raise ValueError(f"expected x of shape [B, C, H, W], got {tuple(x.shape)}")
        if self.training and any(s.dropout > 0 for s in self.levels):
            raise RuntimeError("dropout > 0 in training mode: the native path is inference only -- call model.eval()")
        self._check_cond(class_cond, mapping_cond)
        with torch.cuda.device(x.device):
            xin = _native.f32c(x)
            sig = _native.f32c(sigma).expand(x.shape[0]).contiguous() if sigma.numel() == 1 else _native.f32c(sigma)
            if sig.shape != (x.shape[0],):
                raise ValueError(f"sigma must have shape [{x.shape[0]}], got {tuple(sigma.shape)}")
            eng = self.engine()
            if self.class_emb is not None and not torch.cuda.is_current_stream_capturing():
                eng.check_class_range(class_cond)           # nn.Embedding raises on out-of-range labels (reference :735)
            cond = eng.conditioning(sig, aug_cond, class_cond if self.class_emb is not None else None,
                                    mapping_cond if self.mapping_cond_in_proj is not None else None)
            res = eng.forward(xin, sig, cond, eng.cond_stride, sigma_data, self.resolved_precision(), out=out)
        return res if x.dtype == torch.float32 else res.to(x.dtype)

    def forward(self, x, sigma, aug_cond=None, class_cond=None, mapping_cond=None):
        """F(x, sigma): the raw inner model (reference :721-762)."""
        return self._run(x, sigma, 0.0, aug_cond, class_cond, mapping_cond)

    def denoise(self, x, sigma, sigma_data, aug_cond=None, class_cond=None, mapping_cond=None, out=None):
        """Fused Karras-preconditioned evaluation c_skip x + c_out F(c_in x, sigma) (layers.py:88-90)."""
        return self._run(x, sigma, float(sigma_data), aug_cond, class_cond, mapping_cond, out=out)
