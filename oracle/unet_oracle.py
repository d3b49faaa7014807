"""CPU oracle of the image_v1 U-Net denoiser.  TEST INFRASTRUCTURE ONLY.

A functional (state-dict driven, no nn.Module) fp32 restatement of

    k_diffusion/models/image_v1.py      (ResConvBlock, DBlock, UBlock, MappingNet, ImageDenoiserModelV1.forward)
    k_diffusion/layers.py:116-313       (ConditionedResidualBlock, AdaGN, SelfAttention2d, Downsample2d, Upsample2d,
                                         FourierFeatures, UNet)
    k_diffusion/augmentation.py:92-104  (KarrasAugmentWrapper.forward)

`sd` is the state dict of the bare ImageDenoiserModelV1 (the wrapper's `inner_model.` prefix stripped); `mcfg` is
config['model'] after load_config.  PINNED: tests/test_unet_host.py checks it against the reference outputs that
oracle/make_golden_unet.py recorded.  Every stage can be recorded into `taps` under the names the native engine's
debug taps use (NCHW here, token-major [B, H, W, C] there).
"""
import torch
from torch.nn import functional as F

from .kdiff_oracle import denoiser_forward, fourier_features

GN_EPS = 1e-5
_K1 = torch.tensor([[1 / 8, 3 / 8, 3 / 8, 1 / 8]])                      # layers.py:236-237 'linear'


def gelu(x):
    """nn.GELU() (erf form)"""
    return F.gelu(x)


def ada_gn(sd, p, x, cond, num_groups):
    """layers.py:172-175: group_norm(x) * (weight + 1) + bias, (weight, bias) = mapper(cond).chunk(2)"""
    weight, bias = (cond @ sd[p + "mapper.weight"].T + sd[p + "mapper.bias"]).chunk(2, dim=-1)
    x = F.group_norm(x, num_groups, eps=GN_EPS)
    return torch.addcmul(bias[:, :, None, None], x, weight[:, :, None, None] + 1)


def res_conv_block(sd, p, x, cond, c_in, c_mid, c_out):
    """image_v1.py:15-29 + layers.py:157-159 (Dropout2d is the identity at eval)"""
    h = gelu(ada_gn(sd, p + "main.0.", x, cond, max(1, c_in // 32)))
    h = F.conv2d(h, sd[p + "main.2.weight"], sd[p + "main.2.bias"], padding=1)
    h = gelu(ada_gn(sd, p + "main.4.", h, cond, max(1, c_mid // 32)))
    h = F.conv2d(h, sd[p + "main.6.weight"], sd[p + "main.6.bias"], padding=1)
    skip = F.conv2d(x, sd[p + "skip.weight"]) if c_in != c_out else x
    return h + skip


def self_attention(sd, p, x, cond):
    """layers.py:193-200 with image_v1.py:40-41 (groups max(1, C // 32), heads max(1, C // 64))"""
    n, c, h, w = x.shape
    nh = max(1, c // 64)
    qkv = F.conv2d(ada_gn(sd, p + "norm_in.", x, cond, max(1, c // 32)), sd[p + "qkv_proj.weight"], sd[p + "qkv_proj.bias"])
    qkv = qkv.view([n, nh * 3, c // nh, h * w]).transpose(2, 3)
    q, k, v = qkv.chunk(3, dim=1)
    y = F.scaled_dot_product_attention(q, k, v)
    y = y.transpose(2, 3).contiguous().view([n, c, h, w])
    return x + F.conv2d(y, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def downsample(x):
    """layers.py:259-264: reflect pad 1, depthwise [1,3,3,1]/8 outer product, stride 2"""
    c = x.shape[1]
    k = (_K1.T @ _K1).to(x)
    return F.conv2d(F.pad(x, (1,) * 4, "reflect"), k.expand(c, 1, 4, 4), stride=2, groups=c)


def upsample(x):
    """layers.py:275-280: reflect pad 1, conv_transpose2d with the doubled filter, stride 2, padding 3"""
    c = x.shape[1]
    k1 = _K1 * 2
    k = (k1.T @ k1).to(x)
    return F.conv_transpose2d(F.pad(x, (1,) * 4, "reflect"), k.expand(c, 1, 4, 4), stride=2, padding=3, groups=c)


def mapping(sd, sigma, mapping_cond=None):
    """image_v1.py:136-139: FourierFeatures(log(sigma) / 4) + mapping_cond Linear, then MappingNet (2 x Linear + GELU)"""
    te = fourier_features((sigma.log() / 4)[:, None], sd["timestep_embed.weight"])
    mce = torch.zeros_like(te) if mapping_cond is None else mapping_cond @ sd["mapping_cond.weight"].T
    h = te + mce
    for i in (0, 2):
        h = gelu(h @ sd[f"mapping.{i}.weight"].T + sd[f"mapping.{i}.bias"])
    return h


def _block(sd, p, x, cond, mods, level, tag, taps):
    """ConditionedSequential of (ResConvBlock, [SelfAttention2d]) modules: mods = [(index, kind, c_in, c_mid, c_out)]"""
    for idx, kind, c_in, c_mid, c_out in mods:
        if kind == "res":
            x = res_conv_block(sd, f"{p}{idx}.", x, cond, c_in, c_mid, c_out)
        else:
            x = self_attention(sd, f"{p}{idx}.", x, cond)
        _tap(taps, f"{tag}{level}.{idx}", x)
    return x


def _tap(taps, name, x):
    if taps is not None:
        taps[name] = x.clone()


def block_modules(depth, c_in, c_mid, c_out, attn, first):
    """module list of a DBlock (first = 1, module 0 is the downsample) or UBlock (first = 0), image_v1.py:33-68"""
    mods, idx = [], first
    for i in range(depth):
        my_c_in = c_in if i == 0 else c_mid
        my_c_out = c_mid if i < depth - 1 else c_out
        mods.append((idx, "res", my_c_in, c_mid, my_c_out))
        idx += 1
        if attn:
            mods.append((idx, "attn", my_c_out, my_c_out, my_c_out))
            idx += 1
    return mods, idx


def stage_plan(mcfg):
    """The native engine's debug taps after patch_in, in execution order: tap name -> (tap of its input, op, tap of the DBlock output
    concatenated to the input by a UBlock or None, level whose grid the output is on).  op is ("res" | "attn", state-dict prefix, c_in,
    c_mid, c_out), "down" or "up"; stage_op applies it."""
    depths, channels, attn, n = mcfg["depths"], mcfg["channels"], mcfg["self_attn_depths"], len(mcfg["depths"])
    s0 = mcfg.get("skip_stages", 0)
    stages, skips, prev = {}, {}, "patch_in"
    for i in range(s0, n):
        if i > s0:
            stages[f"d{i}.down"] = (prev, "down", None, i)
            prev = f"d{i}.down"
        mods, _ = block_modules(depths[i], channels[max(0, i - 1)], channels[i], channels[i], attn[i], 1)
        for idx, kind, ci, cm, co in mods:
            stages[f"d{i}.{idx}"] = (prev, (kind, f"u_net.d_blocks.{i}.{idx}.", ci, cm, co), None, i)
            prev = f"d{i}.{idx}"
        skips[i] = prev
    for i in range(n - 1, s0 - 1, -1):
        k = n - 1 - i                                          # u_net.u_blocks holds the UBlocks innermost first
        c_in = channels[i] * 2 if i < n - 1 else channels[i]
        mods, _ = block_modules(depths[i], c_in, channels[i], channels[max(0, i - 1)], attn[i], 0)
        for j, (idx, kind, ci, cm, co) in enumerate(mods):
            stages[f"u{i}.{idx}"] = (prev, (kind, f"u_net.u_blocks.{k}.{idx}.", ci, cm, co), skips[i] if (j == 0 and i < n - 1) else None, i)
            prev = f"u{i}.{idx}"
        if i > s0:
            stages[f"u{i}.up"] = (prev, "up", None, i - 1)
            prev = f"u{i}.up"
    return stages


def stage_op(sd, op, x, cond):
    """one stage of stage_plan applied to its (concatenated) input"""
    if op == "down":
        return downsample(x)
    if op == "up":
        return upsample(x)
    kind, p, c_in, c_mid, c_out = op
    return res_conv_block(sd, p, x, cond, c_in, c_mid, c_out) if kind == "res" else self_attention(sd, p, x, cond)


def level_hw(mcfg, H, W, level):
    """token grid of `level` for an H x W input (patch_size, then one halving per level past skip_stages)"""
    h, w = H // mcfg["patch_size"], W // mcfg["patch_size"]
    for _ in range(mcfg.get("skip_stages", 0), level):
        h, w = h // 2, w // 2
    return h, w


def model_forward(sd, mcfg, x, sigma, mapping_cond=None, taps=None):
    """image_v1.py:135-157 and layers.py:305-312 (UNet.forward)"""
    depths, channels, attn = mcfg["depths"], mcfg["channels"], mcfg["self_attn_depths"]
    ps, skip_stages, n = mcfg["patch_size"], mcfg.get("skip_stages", 0), len(mcfg["depths"])
    cond = mapping(sd, sigma, mapping_cond)
    _tap(taps, "cond", cond)
    if ps > 1:
        x = F.pixel_unshuffle(x, ps)
    x = F.conv2d(x, sd["proj_in.weight"], sd["proj_in.bias"])
    _tap(taps, "patch_in", x)
    skips = []
    for i in range(skip_stages, n):
        if i > skip_stages:
            x = downsample(x)
            _tap(taps, f"d{i}.down", x)
        mods, _ = block_modules(depths[i], channels[max(0, i - 1)], channels[i], channels[i], attn[i], 1)
        x = _block(sd, f"u_net.d_blocks.{i}.", x, cond, mods, i, "d", taps)
        skips.append(x)
    for k, skip in enumerate(reversed(skips)):
        i = n - 1 - k                                          # u_net.u_blocks holds the UBlocks innermost first
        if k > 0:
            x = torch.cat([x, skip], dim=1)
        c_in = channels[i] * 2 if i < n - 1 else channels[i]
        mods, last = block_modules(depths[i], c_in, channels[i], channels[max(0, i - 1)], attn[i], 0)
        x = _block(sd, f"u_net.u_blocks.{k}.", x, cond, mods, i, "u", taps)
        if i > skip_stages:
            x = upsample(x)
            _tap(taps, f"u{i}.up", x)
    x = F.conv2d(x, sd["proj_out.weight"], sd["proj_out.bias"])
    if mcfg.get("has_variance", False):
        x = x[:, :-1]
    if ps > 1:
        x = F.pixel_shuffle(x, ps)
    return x


def augment_forward(sd, mcfg, x, sigma, aug_cond=None, mapping_cond=None, taps=None):
    """augmentation.py:97-104 (KarrasAugmentWrapper) around model_forward"""
    if aug_cond is None:
        aug_cond = x.new_zeros([x.shape[0], 9])
    mapping_cond = aug_cond if mapping_cond is None else torch.cat([aug_cond, mapping_cond], dim=1)
    return model_forward(sd, mcfg, x, sigma, mapping_cond, taps)


def inner_fn(sd, mcfg):
    """the model config.make_model builds: wrapped in KarrasAugmentWrapper when augment_wrapper is set"""
    if mcfg.get("augment_wrapper", True):
        return lambda x, s, **kw: augment_forward(sd, mcfg, x, s, **kw)
    return lambda x, s, **kw: model_forward(sd, mcfg, x, s, **kw)


def make_denoiser(sd, mcfg):
    """Denoiser(inner, sigma_data) as a closure (layers.py:88-90): model(x, sigma, **extra_args)"""
    inner = inner_fn(sd, mcfg)
    sigma_data = mcfg.get("sigma_data", 1.0)
    return lambda x, sigma, **kw: denoiser_forward(inner, x, sigma, sigma_data, **kw)


def strip_prefix(sd):
    """reference state dict (KarrasAugmentWrapper keys `inner_model.*`) -> bare ImageDenoiserModelV1 keys"""
    return {(k[len("inner_model."):] if k.startswith("inner_model.") else k): v for k, v in sd.items()}
