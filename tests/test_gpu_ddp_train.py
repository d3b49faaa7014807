"""Native training under torch DistributedDataParallel (what Accelerate wraps train.py's inner_model and inner_model_ema in) at world
size 2: Denoiser.loss runs the native loss inside DDP's forward and DDP's reducer averages the native backward's gradients.

Each backend's fixture spawns two ranks: gloo with both ranks on cuda:0, and NCCL with one rank per GPU (skipped with fewer than 2 GPUs).
The ranks train the MNIST class-conditional transformer (cfg1) at fp32 and at tf32, and the reference's config_mnist U-Net through the
augment wrapper; each writes what it computed to a file, and the tests below compare the files:

- the DDP gradient equals (g0 + g1) / 2 bit for bit, gi the single-process native gradient of rank i's batch (with 2 ranks DDP's
  division is exact), and it is within the float64 oracle's budget for the two batches together;
- after 5 AdamW steps on param_groups with ema_update (one kdb_ema_update launch per step through both wrappers), both ranks hold the
  same parameters and EMA weights, bit for bit;
- two no_sync() micro-steps and a synced step equal the single-process accumulation of the three;
- the DDP-wrapped EMA model samples on the native CUDA-graph path, bit for bit the unwrapped model's sample;
- a U-Net with skip_stages = 1, whose skipped blocks get no gradient, trains with find_unused_parameters=True."""
import datetime
import json
import os
import socket
import sys
import traceback
from pathlib import Path

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"

pytestmark = pytest.mark.gpu

B = 4            # images per rank
STEPS = 5
CASES = ("cfg1_fp32", "cfg1_tf32", "mnist_unet")
SKIP_CASE = "unet_skip1"


def _config(case):
    if case.startswith("cfg1"):
        return json.loads((GOLDEN / "cfg1_mnist_shapes.json").read_text())["config"]
    if case == "mnist_unet":
        return json.loads((GOLDEN / "unet_configs.json").read_text())["mnist"]["config"]
    return json.loads((GOLDEN / "unet_edges.json").read_text())["patch2_skip1"]["config"]


def build(case, device):
    """(cfg, the model make_model returns, the innermost model, its state dict): the same synth weights on every call and rank"""
    import k_diffusion as K
    from oracle.fixtures import synth_sd
    cfg = K.config.load_config(_config(case))
    outer = K.config.make_model(cfg)
    inner = outer.inner_model if isinstance(outer, K.augmentation.KarrasAugmentWrapper) else outer
    sd = synth_sd({k: list(v.shape) for k, v in inner.state_dict().items()}, 3)
    inner.load_state_dict(sd)
    outer = outer.to(device).eval()
    if case.endswith("tf32"):
        inner.set_train_precision("tf32")
    return cfg, outer, inner, sd


def inputs(cfg, seed, device="cpu"):
    m = cfg["model"]
    H, W = m["input_size"]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, m["input_channels"], H, W, generator=g) * 0.5
    noise = torch.randn(x.shape, generator=g)
    sigma = torch.exp(torch.randn(B, generator=g) * 1.2 - 0.4)
    kw = {}
    if cfg["dataset"]["num_classes"]:
        kw["class_cond"] = torch.randint(0, cfg["dataset"]["num_classes"], (B,), generator=g)
    if m["type"] == "image_v1" and m["augment_wrapper"]:
        kw["aug_cond"] = torch.randn(B, 9, generator=g) * 0.3
    return x.to(device), noise.to(device), sigma.to(device), {k: v.to(device) for k, v in kw.items()}


def _seed(step, rank):
    return 1000 * step + rank


def _grads(inner):
    return {k: p.grad.detach().cpu().clone() for k, p in inner.named_parameters() if p.grad is not None}


def _run_case(case, rank, device, ddp_kw):
    import k_diffusion as K
    from torch.nn.parallel import DistributedDataParallel as DDP
    res = {}

    def wrapped():
        cfg, outer, inner, _ = build(case, device)
        ddp = DDP(outer, device_ids=[device.index], **ddp_kw)
        return cfg, ddp, inner, K.config.make_denoiser_wrapper(cfg)(ddp)

    def solo():
        cfg, outer, inner, _ = build(case, device)
        return inner, K.config.make_denoiser_wrapper(cfg)(outer)

    # one step: the DDP gradient, and this rank's single-process gradient of the same batch
    cfg, ddp, inner, den = wrapped()
    assert den.is_native() and isinstance(den.inner_model, DDP)
    x, noise, sigma, kw = inputs(cfg, _seed(0, rank), device)
    losses = den.loss(x, noise, sigma, **kw)
    assert losses.grad_fn is not None
    losses.mean().backward()
    res["ddp_losses"], res["ddp_grads"] = losses.detach().cpu(), _grads(inner)
    s_inner, s_den = solo()
    s_den.loss(x, noise, sigma, **kw).mean().backward()
    res["solo_grads"] = _grads(s_inner)
    if case == SKIP_CASE:      # a few more steps: DDP finds the unused parameters in every one
        opt = torch.optim.AdamW(K.utils.unwrap_ddp(ddp).param_groups(1e-3), betas=(0.95, 0.999), eps=1e-6, weight_decay=1e-3)
        for step in range(1, 3):
            opt.step()
            opt.zero_grad()
            x, noise, sigma, kw = inputs(cfg, _seed(step, rank), device)
            den.loss(x, noise, sigma, **kw).mean().backward()
        res["late_grads"] = _grads(inner)
        return res

    # STEPS AdamW steps with the EMA update, both models DDP-wrapped as Accelerate wraps them
    cfg, ddp, inner, den = wrapped()
    _, ema_outer, ema_inner, _ = build(case, device)
    ddp_ema = DDP(ema_outer, device_ids=[device.index], **ddp_kw)
    opt = torch.optim.AdamW(K.utils.unwrap_ddp(ddp).param_groups(1e-3), betas=(0.9, 0.95), eps=1e-6, weight_decay=1e-3)
    ema_launches = []
    for step in range(STEPS):
        x, noise, sigma, kw = inputs(cfg, _seed(10 + step, rank), device)
        opt.zero_grad(set_to_none=True)
        den.loss(x, noise, sigma, **kw).mean().backward()
        opt.step()
        before = K._native.launch_breakdown().get("ema", 0)
        K.utils.ema_update(ddp, ddp_ema, 0.9)
        ema_launches.append(K._native.launch_breakdown()["ema"] - before)
    res["ema_launches"] = ema_launches
    res["params"] = {k: v.detach().cpu().clone() for k, v in inner.state_dict().items()}
    res["ema"] = {k: v.detach().cpu().clone() for k, v in ema_inner.state_dict().items()}

    # the EMA model samples through its DDP wrapper on the native graph path, bit for bit as unwrapped
    den_ema = K.config.make_denoiser_wrapper(cfg)(ddp_ema)
    g = torch.Generator().manual_seed(7)
    m = cfg["model"]
    xs = (torch.randn(B, m["input_channels"], *m["input_size"], generator=g) * m["sigma_max"]).to(device)
    sigmas = K.sampling.get_sigmas_karras(6, m["sigma_min"], m["sigma_max"], device=device)
    extra = {"class_cond": kw["class_cond"]} if "class_cond" in kw else {}
    samples = []
    for model in (den_ema, K.config.make_denoiser_wrapper(cfg)(ddp_ema.module)):
        K.sampling.clear_graph_cache()
        replayed = K.sampling._replayed[0]
        with torch.no_grad():
            samples.append(K.sampling.sample_heun(model, xs, sigmas, extra_args=extra, disable=True).cpu())
        res.setdefault("graph_kernels", []).append(K.sampling._replayed[0] - replayed)
    res["sample_equal"] = torch.equal(samples[0], samples[1])
    K.sampling.clear_graph_cache()

    # two no_sync() micro-steps, then a synced one; and the same three batches accumulated by one process
    cfg, ddp, inner, den = wrapped()
    s_inner, s_den = solo()
    for step in range(3):
        batch = inputs(cfg, _seed(20 + step, rank), device)
        s_den.loss(*batch[:3], **batch[3]).mean().backward()
        if step < 2:
            with ddp.no_sync():
                den.loss(*batch[:3], **batch[3]).mean().backward()
            if step == 0:
                res["unsynced_equal"] = all(torch.equal(p.grad, q.grad) for p, q in zip(inner.parameters(), s_inner.parameters()))
        else:
            den.loss(*batch[:3], **batch[3]).mean().backward()
    res["accum_solo"], res["accum_ddp"] = _grads(s_inner), _grads(inner)
    return res


def _worker(rank, world, backend, port, out):
    for p in (str(ROOT), str(ROOT / "k-diffusion_b200"), str(ROOT / "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        device = torch.device("cuda", rank if backend == "nccl" else 0)
        torch.cuda.set_device(device)
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(minutes=5))
        for case in CASES + (SKIP_CASE,):
            ddp_kw = {"find_unused_parameters": True} if case == SKIP_CASE else {}
            torch.save(_run_case(case, rank, device, ddp_kw), Path(out) / f"{case}_{rank}.pt")
        dist.barrier()
        dist.destroy_process_group()
    except BaseException:
        (Path(out) / f"error_{rank}.txt").write_text(traceback.format_exc())
        raise


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module", params=["gloo", "nccl"])
def ranks(request, tmp_path_factory):
    backend = request.param
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL runs one rank per GPU: needs 2 visible GPUs")
    out = tmp_path_factory.mktemp(f"ddp_{backend}")
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, backend, port, str(out))) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(1200)
        if p.is_alive():
            p.kill()
            p.join()
    errors = "".join(e.read_text() for e in sorted(out.glob("error_*.txt")))
    assert all(p.exitcode == 0 for p in procs), f"exit codes {[p.exitcode for p in procs]}\n{errors}"
    return {f.stem: torch.load(f) for f in out.glob("*.pt")}


@pytest.mark.parametrize("case", CASES + (SKIP_CASE,))
def test_ddp_gradient_is_the_mean_of_the_ranks_gradients(ranks, case):
    r0, r1 = ranks[f"{case}_0"], ranks[f"{case}_1"]
    assert set(r0["ddp_grads"]) == set(r0["solo_grads"]) == set(r1["solo_grads"])
    for k, g in r0["ddp_grads"].items():
        assert torch.equal(g, r1["ddp_grads"][k]), k
        assert torch.equal(g, (r0["solo_grads"][k] + r1["solo_grads"][k]) / 2), k


@pytest.mark.parametrize("case", CASES)
def test_ddp_gradient_matches_float64_for_both_batches(ranks, case):
    """within the existing budgets: 8x the oracle's fp32-vs-float64 distance, and at tf32 the tf32 restatement's"""
    r0, r1 = ranks[f"{case}_0"], ranks[f"{case}_1"]
    cfg, _, _, sd = build(case, "cpu")
    parts = [inputs(cfg, _seed(0, r)) for r in range(2)]
    x, noise, sigma = (torch.cat([p[i] for p in parts]) for i in range(3))
    kw = {k: torch.cat([p[3][k] for p in parts]) for k in parts[0][3]}
    gw = torch.full((2 * B,), 1 / (2 * B))          # d mean(losses) / d losses[b] on each rank, averaged by DDP
    got_loss = torch.cat([r0["ddp_losses"], r1["ddp_losses"]])
    from test_gpu_train_tf32 import check_against_restatement
    if case == "mnist_unet":
        from test_gpu_unet_train import check_against_oracle
    else:
        from test_gpu_train import check_against_oracle
    if case == "cfg1_tf32":
        check_against_restatement(cfg, sd, got_loss, r0["ddp_grads"], x, noise, sigma, kw, gw)
    else:
        check_against_oracle(cfg, sd, got_loss, r0["ddp_grads"], x, noise, sigma, kw, gw, device="cuda")


@pytest.mark.parametrize("case", CASES)
def test_adamw_steps_with_ema_keep_the_ranks_identical(ranks, case):
    r0, r1 = ranks[f"{case}_0"], ranks[f"{case}_1"]
    assert r0["ema_launches"] == r1["ema_launches"] == [1] * STEPS      # one kdb_ema_update launch through both DDP wrappers
    for which in ("params", "ema"):
        assert r0[which].keys() == r1[which].keys()
        for k, v in r0[which].items():
            assert torch.equal(v, r1[which][k]), (which, k)
    cfg, _, _, sd = build(case, "cpu")
    assert any(not torch.equal(r0["params"][k], v) for k, v in sd.items())     # the steps did train


@pytest.mark.parametrize("case", CASES)
def test_no_sync_accumulation_equals_single_process(ranks, case):
    r0, r1 = ranks[f"{case}_0"], ranks[f"{case}_1"]
    assert r0["unsynced_equal"] and r1["unsynced_equal"]        # under no_sync() each rank keeps its own gradient
    for k, g in r0["accum_ddp"].items():
        assert torch.equal(g, r1["accum_ddp"][k]), k
        assert torch.equal(g, (r0["accum_solo"][k] + r1["accum_solo"][k]) / 2), k


@pytest.mark.parametrize("case", CASES)
def test_wrapped_ema_model_samples_on_the_native_graph_path(ranks, case):
    for r in (ranks[f"{case}_0"], ranks[f"{case}_1"]):
        assert r["sample_equal"]
        assert r["graph_kernels"][0] > 0 and r["graph_kernels"][0] == r["graph_kernels"][1]


def test_skipped_blocks_get_no_gradient_under_find_unused_parameters(ranks):
    r0, r1 = ranks[f"{SKIP_CASE}_0"], ranks[f"{SKIP_CASE}_1"]
    for r in (r0, r1):
        for grads in (r["ddp_grads"], r["late_grads"]):
            assert grads and not any(k.startswith(("u_net.d_blocks.0.", "u_net.u_blocks.2.")) for k in grads)
    for k, g in r0["late_grads"].items():
        assert torch.equal(g, r1["late_grads"][k]), k
