"""The tf32 training precision on the H100: kdb_wgrad at tf32 (_native.wgrad_tf32) kernel by kernel against float64 sums of its truncated operands, and the whole
model's parameter gradients at tf32 against the tf32 restatement of tests/test_train_tf32_host.py: within a multiple of the restatement's own
fp32-vs-float64 distance, clearly closer to it than to exact arithmetic, with the properties tests/test_gpu_train.py pins at fp32."""
import pytest
import torch

from oracle.make_golden_tf32 import tf32_trunc
from test_gpu_train import CIFAR10, CLASS, LEVELS3, build, inputs, native_grads
from test_train_tf32_host import restated_grads

import k_diffusion as K
from k_diffusion import _native

pytestmark = pytest.mark.gpu


def _want(dy, x, m):
    """float64 dY^T X of the truncated operands, and the bound on fp32 accumulation: 2 m u sum |dY| |X|"""
    a, b = tf32_trunc(dy[:m].cpu()).double(), tf32_trunc(x[:m].cpu()).double()
    return a.T @ b, 2 * m * 2.0 ** -24 * (a.abs().T @ b.abs())


# M at, below and across the first chunk boundary (256 rows for one 64 x 64 tile), N and K tails, many chunks
@pytest.mark.parametrize("M,N,K", [(256, 64, 64), (255, 64, 64), (257, 64, 64), (1000, 96, 40), (5000, 130, 72), (40000, 3, 5),
                                   (20000, 192, 576)])
def test_wgrad_tf32_against_float64_of_truncated_operands(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    dy = torch.randn(M, N + 3, device="cuda", generator=g)[:, 1:N + 1]     # a row stride past N
    x = torch.randn(M, K, device="cuda", generator=g)
    buf = torch.full((N * K + 64,), float("nan"), device="cuda")
    buf[N * K:] = 7.0                                                        # sentinel after the output
    out = _native.wgrad_tf32(dy, x, out=buf[:N * K].view(N, K))
    want, tol = _want(dy, x, M)
    assert not out.isnan().any() and (buf[N * K:] == 7.0).all()
    assert ((out.cpu().double() - want).abs() <= tol + 1e-30).all()
    again = _native.wgrad_tf32(dy, x)
    assert torch.equal(out, again)


@pytest.mark.parametrize("B,hc,wc,Cf,N", [(2, 4, 6, 24, 40), (8, 8, 8, 32, 64), (3, 16, 4, 48, 96)])
def test_wgrad_tf32_merge_gather(B, hc, wc, Cf, N):
    g = torch.Generator(device="cuda").manual_seed(B * hc + Cf)
    fine = torch.randn(B, 2 * hc, 2 * wc, Cf, device="cuda", generator=g)
    M = B * hc * wc
    dy = torch.randn(M, N, device="cuda", generator=g)
    out = _native.wgrad_tf32(dy, fine, merge=(hc, wc))
    gathered = fine.view(B, hc, 2, wc, 2, Cf).permute(0, 1, 3, 2, 4, 5).reshape(M, 4 * Cf)   # TokenMerge: (nh nw e)
    want, tol = _want(dy, gathered, M)
    assert ((out.cpu().double() - want).abs() <= tol + 1e-30).all()
    assert torch.equal(out, _native.wgrad_tf32(dy, gathered))
    # dy rows further apart than N: the merge gather reads them at their stride as the plain route does
    wide = torch.full((M, N + 5), float("nan"), device="cuda")
    wide[:, 2:N + 2] = dy
    assert torch.equal(_native.wgrad_tf32(wide[:, 2:N + 2], fine, merge=(hc, wc)), out)


def _rel(a, b):
    n = b.norm().item()
    return (a.double() - b).norm().item() / n if n > 0 else 0.0


def check_against_restatement(cfg, sd, got_loss, got, x, noise, sigma, kw, gw, simple=False):
    """Each gradient within 8x the tf32 restatement's fp32-vs-float64 distance (plus 1e-6) of its float64 value, and the whole set of
    gradients at least 2x closer to the tf32 restatement than to exact arithmetic (the relative L2 distances summed in quadrature over the
    parameters; on an H100 the ratio is about 2.7 on every model here)"""
    lt64, gt64 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, True, simple)
    _, gt32 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float32, True, simple)
    l64, g64 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, False, simple)
    assert torch.allclose(got_loss.double(), lt64, rtol=1e-4, atol=0)
    assert set(got) == set(gt64)
    to_tf32 = to_exact = 0.0
    for k, want in gt64.items():
        err, ref = _rel(got[k], want), _rel(gt32[k], want)
        assert err <= 8 * ref + 1e-6, f"{k}: rel-L2 {err:.3e} vs the restatement's fp32 distance {ref:.3e}"
        to_tf32 += err ** 2
        to_exact += _rel(got[k], g64[k]) ** 2
    assert to_tf32 * 4 < to_exact, (to_tf32 ** 0.5, to_exact ** 0.5)


@pytest.mark.parametrize("simple", [False, True])
def test_class_conditional_tf32_gradients(simple):
    cfg, inner, sd, model = build({"model": dict(CLASS["model"], loss_config="simple" if simple else "karras"), "dataset": CLASS["dataset"]})
    inner.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 4, 0, classes=[3, 7, 3, 1])
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_restatement(cfg, sd, loss, got, x, noise, sigma, kw, gw, simple)
    assert (got["class_emb.weight"][[0, 2, 4, 5, 6, 8, 9]] == 0).all()


def test_three_levels_with_augment_wrapper_tf32():
    cfg, inner, sd, model = build(LEVELS3, wrap=True)
    model.inner_model.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 2, 1)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_restatement(cfg, sd, loss, got, x, noise, sigma, kw, gw)


def _walk_inputs(cfg, inner, seed):
    """cuda inputs of one engine call on LEVELS3 through the augment wrapper: x, sigma, the conditioning rows and mapping_cond"""
    x, noise, sigma, kw, gw = (t.cuda() if isinstance(t, torch.Tensor) else t for t in inputs(cfg, 2, seed))
    mc = torch.cat([kw["aug_cond"].cuda(), kw["mapping_cond"].cuda()], 1)
    return x, sigma, inner.engine().conditioning(sigma, None, None, mc), mc


def test_train_forward_is_the_forward_of_the_training_walk():
    """The loss's F (kdb_model_train_forward) is bit for bit the out of kdb_model_forward_train at the same precision: at tf32 not the fp32
    forward, at fp32 the fp32 forward"""
    cfg, inner, sd, model = build(LEVELS3, wrap=True)
    x, sigma, cond, mc = _walk_inputs(cfg, inner, 6)
    eng = inner.engine()
    f = eng.train_forward(x, sigma, cond, eng.cond_stride, 0.0, _native.PREC_TF32)
    out = eng.forward_train(x, torch.ones_like(x), sigma, None, None, mc, cond, {}, precision=_native.PREC_TF32)
    assert torch.equal(f, out)
    f32 = eng.forward(x, sigma, cond, eng.cond_stride, 0.0, _native.PREC_FP32)
    assert not torch.equal(f, f32) and (f - f32).norm() < 1e-2 * f32.norm()
    assert torch.equal(eng.train_forward(x, sigma, cond, eng.cond_stride, 0.0, _native.PREC_FP32), f32)
    # the sampling forward ignores the training precision
    inner.set_train_precision("tf32")
    assert torch.equal(inner.engine().forward(x, sigma, cond, eng.cond_stride, 0.0, _native.PREC_FP32), f32)


def test_alternating_precisions_on_one_engine():
    """fp32 and tf32 training walks in turn on one engine, with no rebind between them: each bit for bit that of a fresh engine at its
    precision (the first tf32 call after the finalize builds the tf32 copies, the fp32 calls leave them alone)"""
    cfg, inner, sd, model = build(LEVELS3, wrap=True)
    x, sigma, cond, mc = _walk_inputs(cfg, inner, 11)
    u = torch.randn(x.shape, generator=torch.Generator().manual_seed(12)).cuda()
    params = {k: p for k, p in inner.named_parameters() if p.requires_grad}

    def walk(eng, precision):
        grads = {k: torch.empty(p.shape, device="cuda") for k, p in params.items()}
        return eng.forward_train(x, u, sigma, None, None, mc, cond, grads, precision=precision), grads

    eng = inner.engine()
    order = [_native.PREC_FP32, _native.PREC_TF32, _native.PREC_FP32, _native.PREC_TF32, _native.PREC_TF32, _native.PREC_FP32]
    got = [walk(eng, p) for p in order]
    want = {}
    for p in (_native.PREC_FP32, _native.PREC_TF32):
        fresh = _native.Engine(inner.engine_spec())
        fresh.bind(dict(inner.state_dict(keep_vars=True)))
        want[p] = walk(fresh, p)
    assert not torch.equal(want[_native.PREC_FP32][0], want[_native.PREC_TF32][0])
    for p, (out, grads) in zip(order, got):
        assert torch.equal(out, want[p][0]) and all(torch.equal(g, want[p][1][k]) for k, g in grads.items()), p


def test_two_calls_bit_identical_and_batch_is_sum_of_images_tf32():
    cfg, inner, sd, model = build(LEVELS3, wrap=True)
    inner.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 3, 4)
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    l2, g2 = native_grads(model, inner, x, noise, sigma, kw, gw)
    assert torch.equal(l1, l2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    parts = [native_grads(model, inner, x[i:i + 1], noise[i:i + 1], sigma[i:i + 1], {k: v[i:i + 1] for k, v in kw.items()}, gw[i:i + 1])
             for i in range(3)]
    for k in g1:
        s = sum(p[1][k] for p in parts)
        assert (g1[k] - s).norm() <= 1e-5 * s.norm() + 1e-7, k


def test_adamw_step_on_param_groups_tf32():
    """One AdamW step against the step the tf32 restatement's float64 gradients give.  Adam's first step is lr g / (|g| + eps), about
    lr sign(g), except near |g| ~ eps, where it magnifies the tf32 noise of the gradient; so each parameter's step is held to 2% of its
    L2 norm rather than elementwise (the fp32 suite holds every element to 0.02 lr)."""
    cfg, inner, sd, model = build(CLASS)
    inner.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 4, 5)
    _, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    _, gt64 = restated_grads(cfg, sd, x, noise, sigma, kw, gw, torch.float64, True)
    lr = 2e-4
    opt = torch.optim.AdamW(inner.param_groups(lr), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)
    before = {k: p.detach().clone() for k, p in inner.named_parameters()}
    opt.step()
    ref = {k: torch.nn.Parameter(v.clone().float()) for k, v in sd.items() if k in gt64}
    names = {id(p): k for k, p in inner.named_parameters()}
    groups = [dict(g, params=[ref[names[id(p)]] for p in g["params"]]) for g in inner.param_groups(lr)]
    for k, p in ref.items():
        p.grad = gt64[k].float()
    torch.optim.AdamW(groups, betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3).step()
    for k, p in inner.named_parameters():
        step, want = (p.detach().cpu() - before[k].cpu()), ref[k].detach() - sd[k].float()
        assert (step - want).norm() <= 2e-2 * want.norm(), k


def test_switching_back_to_fp32_gives_the_fp32_bits():
    cfg, inner, sd, model = build(CLASS)
    x, noise, sigma, kw, gw = inputs(cfg, 3, 7)
    l0, g0 = native_grads(model, inner, x, noise, sigma, kw, gw)
    inner.set_train_precision("tf32")
    lt, gt = native_grads(model, inner, x, noise, sigma, kw, gw)
    inner.set_train_precision("fp32")
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    _, fresh, _, fresh_model = build(CLASS)
    l2, g2 = native_grads(fresh_model, fresh, x, noise, sigma, kw, gw)
    assert torch.equal(l0, l1) and torch.equal(l0, l2)
    assert all(torch.equal(g0[k], g1[k]) and torch.equal(g0[k], g2[k]) for k in g0)
    assert not torch.equal(l0, lt) and any(not torch.equal(g0[k], gt[k]) for k in g0)


def test_tf32_copies_follow_the_weights_after_an_update():
    """An optimizer step updates the weights in place; the next loss re-finalizes the engine, and its tf32 copies are those of the updated
    weights: the gradients equal, bit for bit, those of a fresh model built at the updated weights"""
    cfg, inner, sd, model = build(CLASS)
    inner.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 2, 9)
    l0, _ = native_grads(model, inner, x, noise, sigma, kw, gw)
    torch.optim.AdamW(inner.param_groups(1e-2), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3).step()
    l1, g1 = native_grads(model, inner, x, noise, sigma, kw, gw)
    _, fresh, _, fresh_model = build(CLASS)
    fresh.load_state_dict(inner.state_dict())
    fresh.set_train_precision("tf32")
    l2, g2 = native_grads(fresh_model, fresh, x, noise, sigma, kw, gw)
    assert not torch.equal(l0, l1)
    assert torch.equal(l1, l2) and all(torch.equal(g1[k], g2[k]) for k in g1)


def test_cfg1_tf32_gradients():
    """cfg1 (the MNIST class-conditional transformer at 28x28) at tf32 against the restatement"""
    import json
    from pathlib import Path
    spec = json.loads((Path(__file__).resolve().parent / "golden" / "cfg1_mnist_shapes.json").read_text())["config"]
    cfg, inner, sd, model = build(spec)
    inner.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 2, 8)
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_restatement(cfg, sd, loss, got, x, noise, sigma, kw, gw)


def test_cifar10_transformer_tf32_gradients():
    """the CIFAR-10 transformer (two global levels of width 256 and 512, d_head 64) at tf32 against the restatement"""
    cfg, inner, sd, model = build(CIFAR10)
    inner.set_train_precision("tf32")
    x, noise, sigma, kw, gw = inputs(cfg, 2, 13, classes=[10, 6])
    loss, got = native_grads(model, inner, x, noise, sigma, kw, gw)
    check_against_restatement(cfg, sd, loss, got, x, noise, sigma, kw, gw)
