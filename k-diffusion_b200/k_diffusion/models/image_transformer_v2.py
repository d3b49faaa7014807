"""image_transformer_v2 (HDiT) denoiser -- parameter container + native forward.

Constructor signature, spec dataclasses and `state_dict()` layout follow the reference
(k_diffusion/models/image_transformer_v2.py:626-706) so reference checkpoints load unchanged; the
forward pass itself (:721-762) is executed by libkdb200.so.  This module holds no layer logic: it
is a tree of named parameters whose names reproduce the reference keys.  Parameter gradients (training) come from the engine's reverse
walk through `Denoiser.loss`, at fp32 or, after `set_train_precision("tf32")`, with tf32 token-stream GEMMs; `param_groups` returns the
reference's optimizer groups.
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


# Param tags (reference :57-84): "wd" marks the weights that take weight decay, "mapping" the mapping network and the AdaRMSNorm
# projections, which train at a scaled learning rate.
def tag_param(param, tag):
    if not hasattr(param, "_tags"):
        param._tags = set([tag])
    else:
        param._tags.add(tag)
    return param


def tag_module(module, tag):
    for param in module.parameters():
        tag_param(param, tag)
    return module


def apply_wd(module):
    for name, param in module.named_parameters():
        if name.endswith("weight"):
            tag_param(param, "wd")
    return module


def filter_params(function, module):
    for param in module.parameters():
        tags = getattr(param, "_tags", set())
        if function(tags):
            yield param


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


def _ada_linear(width, cond_width):
    """AdaRMSNorm's projection (reference :159-160)"""
    return tag_module(apply_wd(_linear(width, cond_width, zero=True)), "mapping")


def _layer(spec, cond_width):
    kind, _ = _attn_kind(spec.self_attn)
    parts = {}
    if kind != "none":
        d_head = spec.self_attn.d_head
        n_heads = spec.width // d_head
        parts["self_attn"] = _Node(
            norm=_Node(linear=_ada_linear(spec.width, cond_width)),
            qkv_proj=apply_wd(_linear(spec.width * 3, spec.width)),
            scale=torch.full([n_heads], 10.0),
            pos_emb=_Node(freqs=_Buffer(_rope_freqs(d_head, n_heads))),
            out_proj=apply_wd(_linear(spec.width, spec.width, zero=True)),
        )
    parts["ff"] = _Node(
        norm=_Node(linear=_ada_linear(spec.width, cond_width)),
        up_proj=apply_wd(_linear(spec.d_ff * 2, spec.width)),
        down_proj=apply_wd(_linear(spec.width, spec.d_ff, zero=True)),
    )
    return _Node(**parts)


def _level(spec, cond_width):
    return nn.ModuleList([_layer(spec, cond_width) for _ in range(spec.depth)])


class TransformerEngineModel(_native.NativeLossCall, _native.EngineCache, nn.Module):
    """What the transformer models share on top of their parameters: the native engine (a KdbModel of `family`), the precision, and
    the evaluation entry points (the raw model, the Karras-preconditioned denoiser, their JVP / VJP, torch.autograd through x).  A
    subclass sets `levels`, `mapping_spec`, `in_channels`, `out_channels`, `patch_size`, `num_classes`, `mapping_cond_dim`,
    `class_emb`, `mapping_cond_in_proj`, `precision`, `_engines` and the parameter tree whose state-dict keys the engine of its family
    binds."""

    family = _native.FAMILY_ITV2
    kind = "image_transformer_v2"
    dtype_key = "patch_in.proj.weight"      # the parameter whose dtype picks the "auto" precision

    # ------------------------------------------------------------------ engine plumbing
    def engine_spec(self):
        lv = []
        for s in self.levels:
            kind, param = _attn_kind(s.self_attn)
            lv.append(dict(width=s.width, depth=s.depth, d_ff=s.d_ff, attn=kind, d_head=getattr(s.self_attn, "d_head", 0), attn_param=param))
        return dict(levels=lv, in_channels=self.in_channels, out_channels=self.out_channels, patch_size=self.patch_size,
                    mapping_width=self.mapping_spec.width, mapping_depth=self.mapping_spec.depth, mapping_d_ff=self.mapping_spec.d_ff,
                    num_classes=self.num_classes, mapping_cond_dim=self.mapping_cond_dim, family=self.family)

    def engine(self):
        """Native engine with the current parameters bound (rebinds only after the parameters changed)."""
        eng = self._engines.get(None)
        if eng is None:
            eng = self._engines[None] = _native.Engine(self.engine_spec())
        eng.bind(dict(self.state_dict(keep_vars=True)))
        return eng

    def set_precision(self, precision):
        """'fp32' (exact path, parity gate), 'bf16' (tensor-core path) or None/'auto'."""
        self.precision = None if precision in (None, "auto") else precision
        return self

    _TRAIN_PRECISIONS = {None: _native.PREC_FP32, "fp32": _native.PREC_FP32, "float32": _native.PREC_FP32, "tf32": _native.PREC_TF32}

    def set_train_precision(self, precision):
        """The arithmetic of `Denoiser.loss` and its backward: 'fp32' / 'float32' / None (the default, exact fp32) or 'tf32' (every
        token-stream Linear -- qkv, out, up, down, merge and split projections -- with tf32 operands and fp32 accumulation on the tensor
        cores, in the loss's forward, its input gradients and its weight gradients; what an nn.Linear computes under
        torch.backends.cuda.matmul.allow_tf32 = True).  Sampling, `jvp`, `vjp` and autograd through x are not affected."""
        if self.family != _native.FAMILY_ITV2:
            raise NotImplementedError(f"{self.kind}: parameter gradients are built for image_transformer_v2 models only")
        if not (precision is None or isinstance(precision, str)) or precision not in self._TRAIN_PRECISIONS:
            raise ValueError(f"training runs at 'fp32' or 'tf32' (got {precision!r})")
        self.train_precision = self._TRAIN_PRECISIONS[precision]
        return self

    def resolved_precision(self):
        p = flags.resolve_precision(self.precision, self.get_parameter(self.dtype_key).dtype)
        if p in ("tf32", "fp16"):
            raise ValueError(f"the {self.kind} engine runs at fp32 or bf16 ({p} is built for the image_v1 U-Net only)")
        return _native.PREC_BF16 if p == "bf16" else _native.PREC_FP32

    def param_groups(self, base_lr=5e-4, mapping_lr_scale=1 / 3):
        """The reference's four optimizer groups (:708-718): weight decay or not, mapping network (scaled learning rate) or not."""
        wd = filter_params(lambda tags: "wd" in tags and "mapping" not in tags, self)
        no_wd = filter_params(lambda tags: "wd" not in tags and "mapping" not in tags, self)
        mapping_wd = filter_params(lambda tags: "wd" in tags and "mapping" in tags, self)
        mapping_no_wd = filter_params(lambda tags: "wd" not in tags and "mapping" in tags, self)
        return [
            {"params": list(wd), "lr": base_lr},
            {"params": list(no_wd), "lr": base_lr, "weight_decay": 0.0},
            {"params": list(mapping_wd), "lr": base_lr * mapping_lr_scale},
            {"params": list(mapping_no_wd), "lr": base_lr * mapping_lr_scale, "weight_decay": 0.0}
        ]

    def native_loss(self, kind, input, noise, sigma, sigma_data, weight, aug_cond=None, class_cond=None, mapping_cond=None):
        """Per-sample training losses [B] of the Karras-preconditioned denoiser around this model (`_native.LOSS_DENOISER`: reference
        layers.py:76-86 with scales == 1 and per-sample `weight`; `LOSS_SIMPLE`: :107-111), with a grad_fn that reaches every parameter
        requiring grad.  The forward is one engine evaluation and one loss kernel; the backward is one kdb_model_forward_train.  The
        arithmetic is `set_train_precision`'s when the loss is computed (fp32 unless set), for its backward too, whatever `set_precision`
        selected."""
        if kind == _native.LOSS_VARIANCE:
            raise NotImplementedError(f"{self.kind}: DenoiserWithVariance.loss needs the inner model's return_variance output, which the "
                                      "transformers do not have")
        if self.family != _native.FAMILY_ITV2:
            raise NotImplementedError(f"{self.kind}: parameter gradients are built for image_transformer_v2 models only")
        for name, t in (("input", input), ("noise", noise), ("sigma", sigma)):
            if t.requires_grad:
                raise RuntimeError(f"the native loss differentiates the model's parameters only, but {name} requires grad")
        _native.require_cuda(noise)
        if input.ndim != 4 or noise.shape != input.shape:
            raise ValueError(f"expected input and noise of one shape [B, C, H, W], got {tuple(input.shape)} and {tuple(noise.shape)}")
        ev = self.native_eval(input, sigma, aug_cond, class_cond, mapping_cond, precision=_native.PREC_FP32)
        named = [(k, p) for k, p in self.named_parameters() if p.requires_grad]
        keys = tuple(k for k, _ in named)
        return _native.NativeLoss.apply(self, self.engine, ev, kind, _native.f32c(noise), float(sigma_data), weight, keys,
                                        *(p for _, p in named))

    # ------------------------------------------------------------------ forward
    def _check_cond(self, class_cond, mapping_cond):
        _native.require_cond(class_cond, mapping_cond, self.class_emb is not None, self.mapping_cond_in_proj is not None)

    def conditioning(self, sigma, aug_cond=None, class_cond=None, mapping_cond=None):
        """Conditioning table rows for `sigma` [rows] (mapping network + all AdaRMSNorm scales)."""
        self._check_cond(class_cond, mapping_cond)
        return self.engine().conditioning(sigma, aug_cond, class_cond if self.class_emb is not None else None,
                                          mapping_cond if self.mapping_cond_in_proj is not None else None)

    def native_eval(self, x, sigma=None, aug_cond=None, class_cond=None, mapping_cond=None, precision=None):
        """The native front end: validates one evaluation's inputs and returns its `_native.Evaluation` (the bound engine, `precision`
        or, when None, the resolved precision, and the engine's arguments).  Labels are range-checked here, outside stream capture,
        because the conditioning kernel indexes class_emb with them (nn.Embedding raises on out-of-range labels, reference :735)."""
        _native.check_input(x, sigma, self.training and any(s.dropout > 0 for s in self.levels))
        self._check_cond(class_cond, mapping_cond)
        eng = self.engine()
        if self.class_emb is not None and not torch.cuda.is_current_stream_capturing():
            eng.check_class_range(class_cond)
        return _native.Evaluation(eng, self.resolved_precision() if precision is None else precision, x, sigma, aug_cond, class_cond,
                                  mapping_cond, self.class_emb is not None, self.mapping_cond_in_proj is not None)

    def _run(self, x, sigma, sigma_data, aug_cond, class_cond, mapping_cond, out=None, tangent=None, cotangent=None):
        _native.require_cuda(tangent, cotangent)
        derivative = tangent is not None or cotangent is not None
        ev = self.native_eval(x, sigma, aug_cond, class_cond, mapping_cond, _native.PREC_FP32 if derivative else None)
        if not derivative and torch.is_grad_enabled() and x.requires_grad:
            return _autograd_eval(self, ev, x, sigma, sigma_data, aug_cond, mapping_cond, out)
        eng = ev.engine
        if tangent is not None:
            if tangent.shape != x.shape:
                raise ValueError(f"tangent must have the shape of x {tuple(x.shape)}, got {tuple(tangent.shape)}")
            return ev.cast(eng.forward_jvp(ev.x, _native.f32c(tangent), ev.sigma, ev.conditioning(), eng.cond_stride, sigma_data))
        if cotangent is not None:
            return ev.cast(eng.forward_vjp(ev.x, _native.f32c(cotangent), ev.sigma, ev.conditioning(), eng.cond_stride, sigma_data))
        return ev.forward(sigma_data, out)

    def denoise(self, x, sigma, sigma_data, aug_cond=None, class_cond=None, mapping_cond=None, out=None):
        """Fused Karras-preconditioned evaluation c_skip x + c_out F(c_in x, sigma) (layers.py:88-90)."""
        return self._run(x, sigma, float(sigma_data), aug_cond, class_cond, mapping_cond, out=out)

    def jvp(self, x, sigma, v, aug_cond=None, class_cond=None, mapping_cond=None):
        """(F(x, sigma), J_F(x) v): the raw inner model and its forward-mode derivative along `v` with respect to x, in one engine call.
        Always runs on the exact fp32 path, whatever `set_precision` selected (the tangent kernels are fp32 only)."""
        return self._run(x, sigma, 0.0, aug_cond, class_cond, mapping_cond, tangent=v)

    def denoise_jvp(self, x, sigma, v, sigma_data, aug_cond=None, class_cond=None, mapping_cond=None):
        """(D(x, sigma), J_D(x) v) of the Karras-preconditioned evaluation, J_D v = c_skip v + c_out J_F(c_in x) c_in v, in one engine
        call.  Always runs on the exact fp32 path, whatever `set_precision` selected."""
        return self._run(x, sigma, float(sigma_data), aug_cond, class_cond, mapping_cond, tangent=v)

    def vjp(self, x, sigma, u, aug_cond=None, class_cond=None, mapping_cond=None):
        """(F(x, sigma), u^T J_F(x)): the raw inner model and its reverse-mode derivative for the cotangent `u` with respect to x, in one
        engine call.  Always runs on the exact fp32 path, whatever `set_precision` selected (the backward kernels are fp32 only)."""
        return self._run(x, sigma, 0.0, aug_cond, class_cond, mapping_cond, cotangent=u)

    def denoise_vjp(self, x, sigma, u, sigma_data, aug_cond=None, class_cond=None, mapping_cond=None):
        """(D(x, sigma), u^T J_D(x)) of the Karras-preconditioned evaluation, u^T J_D = c_skip u + c_in J_F(c_in x)^T (c_out u), in one
        engine call.  Always runs on the exact fp32 path, whatever `set_precision` selected."""
        return self._run(x, sigma, float(sigma_data), aug_cond, class_cond, mapping_cond, cotangent=u)


class ImageTransformerDenoiserModelV2(TransformerEngineModel):
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

        self.patch_in = _Node(proj=apply_wd(_linear(w0, in_channels * n_patch)))
        self.time_emb = _Node(weight=_Buffer(torch.randn(mw // 2, 1)))            # layers.FourierFeatures(1, mw)
        self.time_in_proj = _linear(mw, mw)
        self.aug_emb = _Node(weight=_Buffer(torch.randn(mw // 2, 9)))             # layers.FourierFeatures(9, mw)
        self.aug_in_proj = _linear(mw, mw)
        self.class_emb = _Node(weight=torch.randn(num_classes, mw)) if num_classes else None
        self.mapping_cond_in_proj = _linear(mw, mapping_cond_dim) if mapping_cond_dim else None
        self.mapping = tag_module(_Node(
            in_norm=_Node(scale=torch.ones(mw)),
            blocks=nn.ModuleList([
                _Node(norm=_Node(scale=torch.ones(mw)), up_proj=apply_wd(_linear(mapping.d_ff * 2, mw)),
                      down_proj=apply_wd(_linear(mw, mapping.d_ff, zero=True)))
                for _ in range(mapping.depth)]),
            out_norm=_Node(scale=torch.ones(mw)),
        ), "mapping")
        self.down_levels = nn.ModuleList([_level(s, mw) for s in levels[:-1]])
        self.up_levels = nn.ModuleList([_level(s, mw) for s in levels[:-1]])
        self.mid_level = _level(levels[-1], mw)
        self.merges = nn.ModuleList([_Node(proj=apply_wd(_linear(b.width, a.width * 4))) for a, b in zip(levels[:-1], levels[1:])])
        self.splits = nn.ModuleList([_Node(proj=apply_wd(_linear(a.width * 4, b.width)), fac=torch.ones(1) * 0.5)
                                     for a, b in zip(levels[:-1], levels[1:])])
        self.out_norm = _Node(scale=torch.ones(w0))
        self.patch_out = _Node(proj=apply_wd(_linear(out_channels * n_patch, w0, zero=True)))

        self.precision = None        # None -> flags.resolve_precision ("auto" unless KDB200_PRECISION is set)
        self._engines = {}

    def forward(self, x, sigma, aug_cond=None, class_cond=None, mapping_cond=None):
        """F(x, sigma): the raw inner model (reference :721-762)."""
        return self._run(x, sigma, 0.0, aug_cond, class_cond, mapping_cond)


class _NativeEval(torch.autograd.Function):
    """torch.autograd through the native engine with respect to x.  The forward is the ordinary engine call at the model's precision (its
    value is bit-identical to a call without grad); the backward is one fp32 forward_vjp at the saved x, sigma and conditioning rows.  At
    bf16 the gradient is therefore that of the fp32 function."""

    @staticmethod
    def forward(ctx, x, model, ev, sigma_data):
        cond = ev.conditioning()
        res = ev.engine.forward(ev.x, ev.sigma, cond, ev.engine.cond_stride, sigma_data, ev.precision)
        ctx.model, ctx.sigma_data, ctx.dtype = model, sigma_data, x.dtype
        ctx.save_for_backward(ev.x, ev.sigma, cond)
        return ev.cast(res)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_out):
        xin, sig, cond = ctx.saved_tensors
        eng = ctx.model.engine()
        _, gx = eng.forward_vjp(xin, _native.f32c(grad_out), sig, cond, eng.cond_stride, ctx.sigma_data)
        return gx.to(ctx.dtype), None, None, None


def _autograd_eval(model, ev, x, sigma, sigma_data, aug_cond, mapping_cond, out):
    """An evaluation whose x requires grad: the gradient reaches x only, so other inputs that require grad are refused, not ignored."""
    for name, t in (("sigma", sigma), ("aug_cond", aug_cond), ("mapping_cond", mapping_cond)):
        if t is not None and t.requires_grad:
            raise RuntimeError(f"the native model is differentiable with respect to x only, but {name} requires grad")
    if out is not None:
        raise RuntimeError("out= cannot be used when x requires grad (the result must carry a grad_fn)")
    return _NativeEval.apply(x, model, ev, sigma_data)
