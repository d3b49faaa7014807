"""Functional restatement of the reference's image_transformer_v1 (k_diffusion/models/image_transformer_v1.py, axial_rope.py) for
tests: the reference's own arithmetic, in the dtype of its inputs, on a state dict in the reference's layout.  TEST INFRASTRUCTURE.

It also states the two folds the native engine runs v1 through (`fold_qknorm`, `fold_rope`), so that tests can check them on the CPU
against the reference form."""
import math

import torch

from . import kdiff_oracle as O

D_HEAD = 64
QK_EPS = 1e-6                     # QKNorm eps (image_transformer_v1.py:109)
MAX_LOG_SCALE = math.log(100.0)   # QKNorm max_scale (:109-112)


def make_axial_pos(h, w, pixel_aspect_ratio=1.0, dtype=torch.float32, device=None):
    """axial_rope.py:43-68 (align_corners False): cell centres of the bounding box whose aspect ratio is w / (h * par), (y, x) [h*w, 2]"""
    ar = w / (h * pixel_aspect_ratio)
    y_min, y_max, x_min, x_max = -1.0, 1.0, -1.0, 1.0
    if ar > 1:
        y_min, y_max = -1 / ar, 1 / ar
    elif ar < 1:
        x_min, x_max = -ar, ar

    def centers(a, b, n):
        e = torch.linspace(a, b, n + 1, dtype=dtype, device=device)
        return (e[:-1] + e[1:]) / 2
    grid = torch.stack(torch.meshgrid(centers(y_min, y_max, h), centers(x_min, x_max, w), indexing="ij"), dim=-1)
    return grid.view(h * w, 2)


def rms_norm(x, scale, eps):
    """rms_norm (:83-87): the statistics in promote_types(x.dtype, float32)"""
    dtype = torch.promote_types(x.dtype, torch.float32)
    mean_sq = torch.mean(x.to(dtype) ** 2, dim=-1, keepdim=True)
    return x * (scale.to(dtype) * torch.rsqrt(mean_sq + eps)).to(x.dtype)


def qk_norm(x, log_scale, eps=QK_EPS):
    """QKNorm.forward (:125-128) with proj_'s clamp (:119-123) applied to a copy: x [..., nh, T, e], log_scale [nh]"""
    s = log_scale.clamp(max=MAX_LOG_SCALE)
    scale = torch.exp(0.5 * s - 0.25 * math.log(x.shape[-1]))
    return rms_norm(x, scale[:, None, None], eps)


def rotate_half(x):
    """axial_rope.py:13-17: the pairs (2j, 2j+1) -> (-x_2j+1, x_2j)"""
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack((-x2, x1), dim=-1).flatten(-2)


def rope_theta(pos, freqs_h, freqs_w):
    """AxialRoPE.get_freqs (axial_rope.py:99-104): pos [T, 2] -> angles [nh, T, e] (each angle twice, interleaved)"""
    th = pos[..., None, None, 0] * freqs_h.exp()
    tw = pos[..., None, None, 1] * freqs_w.exp()
    return torch.cat((th, tw), dim=-1).repeat_interleave(2, dim=-1).transpose(-2, -3)


def apply_rope(x, theta):
    """apply_rotary_emb (axial_rope.py:20-28) with start_index 0 over all e columns"""
    theta = theta.to(x)
    return x * theta.cos() + rotate_half(x) * theta.sin()


def attention_block(sd, p, x, pos, cond):
    """SelfAttentionBlock.forward (:160-173): x [B, T, C]"""
    B, T, C = x.shape
    nh = C // D_HEAD
    xn = O.rms_norm(x, (cond @ sd[p + "norm.linear.weight"].T)[:, None, :] + 1)
    q, k, v = (xn @ sd[p + "qkv_proj.weight"].T).view(B, T, 3, nh, D_HEAD).permute(2, 0, 3, 1, 4).unbind(0)
    theta = rope_theta(pos, sd[p + "pos_emb.freqs_h"], sd[p + "pos_emb.freqs_w"])
    q = apply_rope(qk_norm(q, sd[p + "qk_norm.scale"]), theta)
    k = apply_rope(qk_norm(k, sd[p + "qk_norm.scale"]), theta)
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v)
    return o.transpose(1, 2).reshape(B, T, C) @ sd[p + "out_proj.weight"].T + x


def ff_block(sd, p, x, cond):
    """FeedForwardBlock.forward (:185-192)"""
    xn = O.rms_norm(x, (cond @ sd[p + "norm.linear.weight"].T)[:, None, :] + 1)
    return O.linear_geglu(xn, sd[p + "up_proj.weight"]) @ sd[p + "down_proj.weight"].T + x


def model_forward(sd, mcfg, x, sigma, aug_cond=None, class_cond=None):
    """ImageTransformerDenoiserModelV1.forward (:317-344).  `mcfg` is config['model'] after load_config (depth, patch_size)."""
    ps = mcfg["patch_size"]
    ph, pw = (ps, ps) if isinstance(ps, int) else ps
    B, c, H, W = x.shape
    h, w = H // ph, W // pw
    # Patching (:217-226): '... c (h i) (w j) -> ... (h w) (c i j)', positions with pixel_aspect_ratio = patch_h / patch_w
    t = x.view(B, c, h, ph, w, pw).permute(0, 2, 4, 1, 3, 5).reshape(B, h * w, c * ph * pw)
    pos = make_axial_pos(h, w, ph / pw, dtype=x.dtype, device=x.device)
    t = t @ sd["in_proj.weight"].T
    if class_cond is None and "class_emb.weight" in sd:
        raise ValueError("class_cond must be specified if num_classes > 0")
    c_noise = torch.log(sigma) / 4
    emb = O.fourier_features(c_noise[..., None], sd["time_emb.weight"]) @ sd["time_in_proj.weight"].T
    aug = t.new_zeros([B, 9]) if aug_cond is None else aug_cond
    emb = emb + O.fourier_features(aug, sd["aug_emb.weight"]) @ sd["aug_in_proj.weight"].T
    if "class_emb.weight" in sd:
        emb = emb + sd["class_emb.weight"][class_cond]
    cond = O.mapping_network(sd, emb)
    for i in range(mcfg["depth"]):
        t = attention_block(sd, f"blocks.{i}.self_attn.", t, pos, cond)
        t = ff_block(sd, f"blocks.{i}.ff.", t, cond)
    t = O.rms_norm(t, sd["out_norm.scale"]) @ sd["out_proj.weight"].T
    # Unpatching (:239-243): '... (h w) (c i j) -> ... c (h i) (w j)'
    co = t.shape[-1] // (ph * pw)
    return t.view(B, h, w, co, ph, pw).permute(0, 3, 1, 4, 2, 5).reshape(B, co, H, W)


def make_denoiser(sd, mcfg):
    """Denoiser(inner_model, sigma_data) as a closure: model(x, sigma, **extra_args)."""
    sigma_data = mcfg.get("sigma_data", 1.0)

    def model(x, sigma, **kw):
        return O.denoiser_forward(lambda xi, s, **k2: model_forward(sd, mcfg, xi, s, **k2), x, sigma, sigma_data, **kw)
    return model


# ---------------------------------------------------------------------------------------------- the engine's folds

def fold_qknorm(log_scale, e=D_HEAD):
    """(cosine-sim scale per head, eps on the sum of squares) that equal QKNorm + SDPA's 1/sqrt(e)"""
    return torch.exp(log_scale.clamp(max=MAX_LOG_SCALE)), e * QK_EPS


def head_permutation(e=D_HEAD):
    """new column j <- old 2j, new column j + e/2 <- old 2j + 1"""
    return torch.cat([torch.arange(0, e, 2), torch.arange(1, e, 2)])


def fold_rope(freqs_h, freqs_w):
    """the engine's QkRope frequency table [nh, e/2] (R = e): y frequencies, then x"""
    return torch.cat([freqs_h.exp(), freqs_w.exp()], dim=-1)


def engine_qk(q, pos, scale, eps, table):
    """the engine's cosine sim + half-split RoPE of R = e columns (QkRope): q [..., nh, T, e] in the permuted column order"""
    e = q.shape[-1]
    q = q * (torch.sqrt(scale)[:, None, None] * torch.rsqrt((q * q).sum(-1, keepdim=True) + eps))
    nf = e // 4
    th = torch.cat([pos[:, 0:1] * table[:, None, :nf], pos[:, 1:2] * table[:, None, nf:]], dim=-1)   # [nh, T, e/2]
    c, s = th.cos(), th.sin()
    x1, x2 = q[..., :e // 2], q[..., e // 2:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)
