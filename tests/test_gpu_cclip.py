"""Centered clipping on the GPU: K23 (``cclip_aggregate_slots``) against the CPU oracle (odd rows, padded banks, a 4-byte
aligned arena, up to 256 clients, the distance mask, several iterations from a nonzero center, every server optimizer),
bit-exactness when nothing is clipped, run-to-run bit identity, the binding's checks, the fused round kernel's
centered-clipping phase against the oracle and the generic executor over every cluster size and warps-per-pair setting with
the state carried across rounds and launches, CUDA-graph replay, capacity routing and the Byzantine scenarios."""
import copy

import numpy as np
import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.ops.server_opt import SlotServerOpt
from test_cclip import ATTACKED_MEAN_MAX, CCLIP_KW, CCLIP_MIN, attacked_honest_acc
from test_gpu_small_round import make_state, to_cuda
from test_robust_agg import BYZ, BYZ_KW, _same

pytestmark = pytest.mark.gpu


def _case(C, M, P, stride, seed=1, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, stride, generator=g)
    up = bank[None, :, :P] + scale * torch.randn(C, M, P, generator=g)
    n = (torch.rand(C, M, generator=g) * 4).floor()
    n[0] = 1.0
    if M > 1:
        n[:, -1] = 0                       # the last slot has no participant: θ and h stay
    center = 0.1 * scale * torch.randn(M, P, generator=g)
    return bank, up, n, center


def _close(a, b, rtol=1e-5, atol=1e-6):
    return torch.allclose(a.double(), b.double(), rtol=rtol, atol=atol, equal_nan=True)


def _run_both(bank, up, n, center, P, tau, iters, mask=None, cp=None):
    want, want_h = bank.clone(), center.clone()
    cnt = ref.cclip_aggregate_slots_(want[:, :P], up, n, want_h, tau, iters, mask)
    gb, gh = bank.cuda(), center.cuda()
    got = ops.cclip_aggregate_slots_(gb[:, :P], up.cuda() if cp is None else cp, n.cuda(), gh, tau, iters, None,
                                     None if mask is None else mask.cuda())
    torch.cuda.synchronize()
    return (gb.cpu(), gh.cpu(), got.cpu()), (want, want_h, cnt)


@pytest.mark.parametrize("iters", [1, 5])
@pytest.mark.parametrize("C,M,P,stride,masked", [
    (1, 2, 37, 37, False), (2, 2, 64, 64, True), (3, 2, 37, 40, False), (7, 3, 1001, 1001, True), (7, 3, 1003, 1024, False),
    (100, 2, 4096, 4096, True), (256, 2, 515, 520, False), (256, 1, 2048, 2048, True),
])
def test_k23_matches_reference(C, M, P, stride, masked, iters):
    bank, up, n, center = _case(C, M, P, stride)
    mask = (torch.arange(P) % 9 != 4) if masked else None
    tau = 0.3 * float(np.sqrt(P))          # clips part of the rows
    (gb, gh, got), (want, want_h, cnt) = _run_both(bank, up, n, center, P, tau, iters, mask)
    assert _close(gb, want) and _close(gh, want_h), ((gb - want).abs().max(), (gh - want_h).abs().max())
    assert torch.equal(gb[:, P:], bank[:, P:]) and torch.equal(got, cnt)
    if M > 1:                              # the slot without participants keeps θ and h
        assert torch.equal(gb[-1], bank[-1]) and torch.equal(gh[-1], center[-1])
    # a radius above every distance clips nothing: then the result is bit-identical
    (gb, gh, _), (want, want_h, _) = _run_both(bank, up, n, center, P, 1e30, iters, mask)
    assert _same(gb, want) and _same(gh, want_h)


def test_k23_misaligned_arena_scalar_path_and_edge_cases():
    C, M, P = 9, 3, 203
    bank, up, n, center = _case(C, M, P, P, seed=5)
    n[:, :2] = 1.0
    flat = torch.zeros(C * M * P + 1)
    flat[1:] = up.reshape(-1)
    cp = flat.cuda()[1:].view(C, M, P)                    # 4-byte aligned only
    up[2, 0, 7] = float("inf")                             # slot 0: dropped (s = 0)
    cp[2, 0, 7] = float("inf")
    up[4, 1, 3] = float("nan")                             # slot 1: NaN in θ and h
    cp[4, 1, 3] = float("nan")
    for iters in (1, 4):
        (gb, gh, _), (want, want_h, _) = _run_both(bank, up, n, center, P, 2.0, iters, None, cp)
        assert _close(gb, want) and _close(gh, want_h)
        assert torch.isfinite(gb[0]).all() and torch.isfinite(gh[0]).all()
        assert (gb[1].view(torch.int32) == 0x7FC00000).all() and (gh[1].view(torch.int32) == 0x7FC00000).all()


@pytest.mark.parametrize("kind", ["sgd", "adam", "adagrad", "yogi"])
def test_k23_with_server_optimizer(kind):
    C, M, P = 9, 3, 1001
    bank, up, n, center = _case(C, M, P, P, seed=4)
    mask = torch.arange(P) % 7 != 0
    hp = dict(lr=0.05, momentum=0.9 if kind == "sgd" else 0.0, eps=1e-3)
    rule = ("centered_clip", 0.1, 8.0, 2)
    cpu_so = SlotServerOpt(kind, M, P, "cpu", mask=mask, **hp)
    gpu_so = SlotServerOpt(kind, M, P, "cuda", mask=mask, **hp)
    cpu, gpu = bank.clone(), bank.cuda()
    ch, gh = center.clone(), center.cuda()
    for _ in range(2):
        ops.cluster_aggregate_(cpu, up, n, cpu_so, rule, mask=mask, center=ch)
        ops.cluster_aggregate_(gpu, up.cuda(), n.cuda(), gpu_so, rule, mask=mask.cuda(), center=gh)
    torch.cuda.synchronize()
    assert torch.equal(gpu_so.step.cpu(), cpu_so.step) and gpu_so.step.tolist() == [2, 2, 0]
    assert torch.allclose(gpu.cpu(), cpu, rtol=1e-4, atol=1e-5), (gpu.cpu() - cpu).abs().max()
    assert torch.allclose(gh.cpu(), ch, rtol=1e-4, atol=1e-5)


def test_k23_bit_identical_across_launches():
    bank, up, n, center = _case(64, 2, 100_003, 100_008, seed=7)
    up, n = up.cuda(), n.cuda()
    outs = []
    for _ in range(3):
        gb, gh = bank.cuda(), center.cuda()
        ops.cclip_aggregate_slots_(gb[:, :100_003], up, n, gh, 50.0, 3)
        outs.append((gb, gh))
    torch.cuda.synchronize()
    for gb, gh in outs[1:]:
        assert _same(outs[0][0], gb) and _same(outs[0][1], gh)


def test_binding_rejects_bad_input():
    ext = ops._ext.load()
    th, cp, n = torch.zeros(2, 8, device="cuda"), torch.zeros(3, 2, 8, device="cuda"), torch.ones(3, 2, device="cuda")
    h = torch.zeros(2, 8, device="cuda")
    for tau, it in [(1.0, 0), (1.0, 101), (0.0, 1), (-1.0, 1), (float("nan"), 1), (float("inf"), 1), (1e-46, 1), (1e39, 1)]:
        with pytest.raises(RuntimeError):
            ext.cclip_aggregate_slots(th, cp, n, h, tau, it, 0, 0.0, 0.0, 1e-8, None, None, None, None, None)
    with pytest.raises(RuntimeError):
        ext.cclip_aggregate_slots(th, cp, n, h, 1.0, 1, 2, 0.1, 0.0, 1e-8, None, None, None, None, None)   # adam without state
    with pytest.raises(RuntimeError):
        ext.cclip_aggregate_slots(th, cp, n, torch.zeros(2, 7, device="cuda"), 1.0, 1, 0, 0.0, 0.0, 1e-8, None, None, None, None,
                                  None)
    with pytest.raises(RuntimeError):
        ext.cclip_aggregate_slots(th, cp, n, h, 1.0, 1, 0, 0.0, 0.0, 1e-8, None, None, None, None,
                                  torch.ones(7, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.fed_round_small(dict(to_cuda(make_state()), aggregation_rule="centered_clip", cclip_iters=0), 1)
    with pytest.raises(ValueError):
        ops.cluster_aggregate_(th, cp, n, None, ("centered_clip", 0.1, 1.0, 1))


def _cc(st, tau=0.05, iters=3, seed=2):
    M, P = st["theta"].shape
    h = 0.01 * torch.randn(M, P, generator=torch.Generator().manual_seed(seed))
    return dict(st, aggregation_rule="centered_clip", cclip_tau=tau, cclip_iters=iters, cclip_center=h)


SHAPES = [dict(), dict(kind="lr", hid=0), dict(din=2, hid=4), dict(kind="fnn", din=4, hid=8, dout=3), dict(C=37, M=4)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("wpp", [1, 2, 4])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_fused_matches_oracle_and_generic(shape, wpp, G):
    st = dict(_cc(make_state(**shape)), cluster=G, warps_per_pair=wpp)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 3)                               # the state carried over three rounds of one launch ...
    ref.fed_round_small(st, 3)
    ops.fed_round_small(g, 2)                               # ... and into a second launch
    ref.fed_round_small(st, 2)
    torch.cuda.synchronize()
    assert torch.allclose(g["theta"].cpu(), st["theta"], rtol=1e-4, atol=1e-5), (g["theta"].cpu() - st["theta"]).abs().max()
    assert torch.allclose(g["cclip_center"].cpu(), st["cclip_center"], rtol=1e-4, atol=1e-5)
    # one round on the kernel's own uploads: its aggregation equals K23 (and the oracle) applied to them
    C, M, P = st["X"].shape[1], *st["theta"].shape
    g["client_out"] = torch.zeros(C, M, P, device="cuda")
    theta0, h0 = g["theta"].clone(), g["cclip_center"].clone()
    ops.fed_round_small(g, 1)
    torch.cuda.synchronize()
    up = g["client_out"]
    sel = (up != 0).any(-1).float()
    k23, k23h = theta0.clone(), h0.clone()
    ops.cclip_aggregate_slots_(k23, up, sel, k23h, 0.05, 3)
    want, want_h = theta0.cpu().clone(), h0.cpu().clone()
    ref.cclip_aggregate_slots_(want, up.cpu(), sel.cpu(), want_h, 0.05, 3)
    assert _close(g["theta"].cpu(), k23.cpu()) and _close(g["theta"].cpu(), want)
    assert _close(g["cclip_center"].cpu(), k23h.cpu()) and _close(g["cclip_center"].cpu(), want_h)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_fused_with_server_optimizer(kind):
    from test_server_opt import with_server_opt
    from test_gpu_server_opt import _compare
    st = with_server_opt(_cc(make_state()), kind)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 3)
    ref.fed_round_small(st, 3)
    torch.cuda.synchronize()
    _compare(g, st)
    assert torch.allclose(g["cclip_center"].cpu(), st["cclip_center"], rtol=1e-4, atol=1e-5)


def test_fused_is_bit_identical_across_runs_and_launch_splits():
    st = dict(_cc(make_state(C=12)), cluster=4)
    one, again, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    ops.fed_round_small(again, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    assert _same(one["theta"], again["theta"]) and _same(one["theta"], three["theta"])
    assert _same(one["cclip_center"], again["cclip_center"]) and _same(one["cclip_center"], three["cclip_center"])


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, aggregation_rule="centered_clip", cclip_tau=0.05, cclip_iters=2)
    d.update(kw)
    return DriftSim(make_args(**d), device="cuda", sink=MetricsSink())


def test_fused_and_generic_engines_agree_over_two_time_steps():
    a, b = _sim(), _sim()
    b.algo.fused_ok = lambda: False
    from feddrift_b200.ops import small_round
    n0 = small_round.LAUNCH_COUNT["fed_round_small"]
    a.run(end_iteration=2)
    assert small_round.LAUNCH_COUNT["fed_round_small"] > n0
    b.run(end_iteration=2)
    torch.cuda.synchronize()
    assert torch.allclose(a.bank.theta, b.bank.theta, rtol=1e-4, atol=1e-5), (a.bank.theta - b.bank.theta).abs().max()
    assert torch.allclose(a.bank.cclip_center, b.bank.cclip_center, rtol=1e-4, atol=1e-5)
    assert bool(a.bank.cclip_center.any())


def test_round_graph_replay_matches_non_graph_path():
    def make():
        sim = _sim(client_num_per_round=5)
        sim.run_time_step(0, rounds=3)
        sim.begin_time_step(1)
        sim.run_rounds(1)
        sim.args.rounds_per_launch = 1
        return sim

    a, b = make(), make()
    ha, hb = a.make_host_round_inputs(), b.make_host_round_inputs()
    h_before, th_before = a.bank.cclip_center.clone(), a.bank.theta.clone()
    assert bool(h_before.any())
    build, seen = a._build_round_graph, {}

    def build_and_look(host):                              # the warm-up launch is undone: building advances nothing
        g = build(host)
        torch.cuda.synchronize()
        seen["h"], seen["theta"] = a.bank.cclip_center.clone(), a.bank.theta.clone()
        return g

    a._build_round_graph = build_and_look
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert _same(seen["h"], h_before) and _same(seen["theta"], th_before)
    assert _same(a.bank.theta, b.bank.theta) and _same(a.bank.cclip_center, b.bank.cclip_center)


def test_fits_routes_and_cfg2_runs_fused():
    from feddrift_b200.experiments.configs import CONFIGS
    from feddrift_b200.ops import small_round
    # fnn 4-8-3 (P = 67, 8 warps): centered clipping needs the geometric median's C·69 + 4 ≤ 8·33·67 (C ≤ 256)
    assert small_round.fits("fnn", 4, 8, 3, 256, 2, 0, rule="centered_clip")
    assert not small_round.fits("fnn", 4, 8, 3, 257, 2, 0, rule="centered_clip")
    assert small_round.fits("fnn", 4, 8, 3, 257, 2, 0, robust=True)
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    cfg = dict(CONFIGS["cfg2c_sea_fnn_100clients_cclip_feddrift"], comm_round=2, total_train_iteration=2)
    s = DriftSim(make_args(**cfg), device="cuda", sink=MetricsSink())
    s.begin_time_step(0)
    assert s._use_fused()
    n0 = small_round.LAUNCH_COUNT["fed_round_small"]
    s.run_rounds(2)
    assert small_round.LAUNCH_COUNT["fed_round_small"] > n0 and torch.isfinite(s.bank.theta).all()
    assert bool(s.bank.cclip_center.any())
    # SEA fnn (P = 38, 12 warps): 400 clients pass the ranking's 2·C ≤ 33·P but need 400·40 + 4 > 12·33·38 floats, so the
    # generic executor (K23) takes them
    spec = s.spec
    assert small_round.fits(spec["kind"], spec["in"], spec["hidden"], spec["out"], 400, 4, 0, rule="median")
    assert not small_round.fits(spec["kind"], spec["in"], spec["hidden"], spec["out"], 400, 4, 0, rule="centered_clip")
    big = DriftSim(make_args(client_num_in_total=400, sample_num=20, comm_round=1, total_train_iteration=1, epochs=1,
                             aggregation_rule="centered_clip"), device="cuda", sink=MetricsSink())
    big.begin_time_step(0)
    assert big.spec is not None and not big._use_fused()
    n0 = small_round.LAUNCH_COUNT["fed_round_small"]
    big.run_rounds(1)
    assert small_round.LAUNCH_COUNT["fed_round_small"] == n0 and torch.isfinite(big.bank.theta).all()
    assert bool(big.bank.cclip_center.any())


def test_generic_executor_route():
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    sim = DriftSim(make_args(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                             concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                             total_train_iteration=2, epochs=2, aggregation_rule="centered_clip", cclip_tau=0.5, cclip_iters=2),
                   device="cuda", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    sim.run_rounds(1)
    theta0, h0 = sim.bank.theta.cpu().clone(), sim.bank.cclip_center.cpu().clone()
    sim.run_rounds(1)
    torch.cuda.synchronize()
    want, want_h = theta0.clone(), h0.clone()
    mask = None if sim.defense_mask is None else sim.defense_mask.cpu()
    ref.cclip_aggregate_slots_(want, sim.clients.params.cpu(), sim.clients.n.cpu(), want_h, 0.5, 2, mask)
    assert _close(sim.bank.theta.cpu(), want, rtol=1e-4, atol=1e-5) and _close(sim.bank.cclip_center.cpu(), want_h, rtol=1e-4,
                                                                                atol=1e-5)


def test_byzantine_sign_flip_on_the_fused_kernel():
    from feddrift_b200.ops import small_round
    n0 = small_round.LAUNCH_COUNT["fed_round_small"]
    cc, sim = attacked_honest_acc("centered_clip", "sign_flip", "cuda")
    assert sim._use_fused() and small_round.LAUNCH_COUNT["fed_round_small"] > n0
    mean, _ = attacked_honest_acc("mean", "sign_flip", "cuda")
    assert cc >= CCLIP_MIN and mean <= ATTACKED_MEAN_MAX and np.isfinite(cc), (cc, mean)


def test_byzantine_alie_on_the_generic_executor():
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    sim = DriftSim(make_args(aggregation_rule="centered_clip", attack_type="alie", attack_clients=BYZ, attack_scale=1.0,
                             **CCLIP_KW, **BYZ_KW), device="cuda", sink=MetricsSink())
    sim.run()
    assert not sim._use_fused()                            # ALIE needs every upload of a slot: the generic executor runs it
    acc = sim.sink.series("Test/AccHonest")[-1]
    assert np.isfinite(acc) and acc >= CCLIP_MIN, acc
