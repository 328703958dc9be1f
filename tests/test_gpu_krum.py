"""Multi-Krum on the GPU: K21 (``krum_aggregate_slots``) against the CPU oracle, bit for bit on separated data (odd rows,
misaligned arenas, padded banks, up to 256 clients, the distance mask, n = 1 and 2, a ResNet-18-sized arena), every
server optimizer, run-to-run bit identity, the binding's checks, the fused round kernel's Multi-Krum phase against the
oracle, K21 and the generic executor over every cluster size and warps-per-pair setting, CUDA-graph replay, capacity
routing and the Byzantine scenario."""
import copy

import numpy as np
import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.ops.server_opt import SlotServerOpt
from test_gpu_small_round import make_state, to_cuda
from test_krum import KRUM_MIN, krum_honest_test_acc
from test_robust_agg import MEAN_MAX, _same, honest_test_acc

pytestmark = pytest.mark.gpu


def _case(C, M, P, stride, seed=1):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, stride, generator=g)
    scale = 1.0 + torch.rand(C, 1, 1, generator=g) * 3   # spread the scores apart
    up = torch.randn(C, M, P, generator=g) * scale + torch.randn(1, M, P, generator=g)
    n = (torch.rand(C, M, generator=g) * 4).floor()
    n[0] = 1.0
    if M > 1:
        n[:, -1] = 0                       # the last slot has no participant
    return bank, up, n


@pytest.mark.parametrize("C,M,P,stride,masked,f,m", [
    (1, 2, 37, 37, False, 1, 1), (2, 2, 64, 64, False, 0, 1), (2, 2, 64, 64, False, 0, 2), (3, 2, 37, 40, False, 1, 2),
    (7, 3, 1001, 1001, True, 1, 3), (7, 3, 1003, 1024, False, 2, 1), (10, 2, 4096, 4096, True, 1, 20),
    (100, 2, 4096, 4096, True, 3, 5), (256, 2, 515, 520, False, 10, 3), (256, 1, 2048, 2048, True, 0, 1),
])
def test_k21_matches_reference_bitwise(C, M, P, stride, masked, f, m):
    bank, up, n = _case(C, M, P, stride)
    mask = (torch.arange(P) % 9 != 4) if masked else None
    want = bank.clone()
    cnt = ref.krum_aggregate_slots_(want[:, :P], up, n, f, m, mask)
    gb = bank.cuda()
    got = ops.krum_aggregate_slots_(gb[:, :P], up.cuda(), n.cuda(), f, m, None, None if mask is None else mask.cuda())
    torch.cuda.synchronize()
    assert _same(gb.cpu(), want), (gb.cpu() - want).abs().max()
    assert torch.equal(gb.cpu()[:, P:], bank[:, P:]) and torch.equal(gb.cpu()[-1], want[-1])
    assert torch.equal(got.cpu(), cnt)


def test_k21_misaligned_arena_scalar_path_and_edge_cases():
    C, M, P = 9, 2, 203
    bank, up, n = _case(C, M, P, P, seed=5)
    n[:] = 1
    flat = torch.zeros(C * M * P + 1)
    flat[1:] = up.reshape(-1)
    cp = flat.cuda()[1:].view(C, M, P)                    # 4-byte aligned only
    up[2, 0, 7] = float("inf")
    cp[2, 0, 7] = float("inf")
    up[5, 1, 0] = float("nan")
    cp[5, 1, 0] = float("nan")
    for m in (1, 3):
        want = bank.clone()
        ref.krum_aggregate_slots_(want, up, n, 1, m)
        gb = bank.cuda()
        ops.krum_aggregate_slots_(gb, cp, n.cuda(), 1, m)
        torch.cuda.synchronize()
        assert _same(gb.cpu(), want) and torch.isfinite(gb.cpu()).all()
    gb = bank.cuda()                                      # m_eff = n: the non-finite rows propagate, as in the oracle
    want = bank.clone()
    ref.krum_aggregate_slots_(want, up, n, 1, 9)
    ops.krum_aggregate_slots_(gb, cp, n.cuda(), 1, 9)
    got = gb.cpu()                                        # a NaN's payload may differ: compare where the oracle is a number
    assert torch.equal(torch.isnan(got), torch.isnan(want)) and torch.isnan(want).any()
    assert _same(got[~torch.isnan(want)], want[~torch.isnan(want)])
    gb = bank.cuda()                                      # n = 1: the upload itself
    ops.krum_aggregate_slots_(gb, up[3:4].cuda(), torch.ones(1, M).cuda(), 1, 4)
    assert _same(gb.cpu(), up[3])
    two = bank.clone()                                    # n = 2: k = 1, both scores equal, m = 1 takes the lower client
    ref.krum_aggregate_slots_(two, up[:2], torch.ones(2, M), 0, 1)
    gb = bank.cuda()
    ops.krum_aggregate_slots_(gb, up[:2].cuda(), torch.ones(2, M).cuda(), 0, 1)
    assert _same(gb.cpu(), two) and _same(two, up[0])


@pytest.mark.parametrize("kind", ["sgd", "adam", "adagrad", "yogi"])
def test_k21_with_server_optimizer(kind):
    C, M, P = 9, 3, 1001
    bank, up, n = _case(C, M, P, P, seed=4)
    mask = torch.arange(P) % 7 != 0
    hp = dict(lr=0.05, momentum=0.9 if kind == "sgd" else 0.0, eps=1e-3)
    rule = ("multi_krum", 0.1, 1, 2)
    cpu_so = SlotServerOpt(kind, M, P, "cpu", mask=mask, **hp)
    gpu_so = SlotServerOpt(kind, M, P, "cuda", mask=mask, **hp)
    cpu, gpu = bank.clone(), bank.cuda()
    for _ in range(2):
        ops.cluster_aggregate_(cpu, up, n, cpu_so, rule, mask=mask)
        ops.cluster_aggregate_(gpu, up.cuda(), n.cuda(), gpu_so, rule, mask=mask.cuda())
    torch.cuda.synchronize()
    assert torch.equal(gpu_so.step.cpu(), cpu_so.step) and gpu_so.step.tolist() == [2, 2, 0]
    assert torch.allclose(gpu.cpu(), cpu, rtol=1e-4, atol=1e-5), (gpu.cpu() - cpu).abs().max()


def test_k21_bit_identical_across_launches():
    bank, up, n = _case(64, 2, 100_003, 100_008, seed=7)
    up, n = up.cuda(), n.cuda()
    outs = []
    for _ in range(3):
        gb = bank.cuda()
        ops.krum_aggregate_slots_(gb[:, :100_003], up, n, 3, 4)
        outs.append(gb)
    torch.cuda.synchronize()
    assert _same(outs[0], outs[1]) and _same(outs[0], outs[2])


def test_k21_resnet18_arena():
    P, C, M = 11_689_512, 32, 2
    g = torch.Generator(device="cuda").manual_seed(9)
    bank = torch.randn(M, P + 8, device="cuda", generator=g)
    up = torch.randn(C, M, P, device="cuda", generator=g) * (1.0 + torch.arange(C, device="cuda")[:, None, None] / 16)
    n = torch.ones(C, M, device="cuda")
    n[3, 1] = 0
    want = bank.clone()
    ref.krum_aggregate_slots_(want[:, :P], up, n, 4, 3)     # the oracle on device tensors (same definition)
    gb = bank.clone()
    ops.krum_aggregate_slots_(gb[:, :P], up, n, 4, 3)
    torch.cuda.synchronize()
    assert _same(gb, want), (gb - want).abs().max()


def test_binding_rejects_bad_input():
    ext = ops._ext.load()
    th, cp, n = torch.zeros(2, 8, device="cuda"), torch.zeros(3, 2, 8, device="cuda"), torch.ones(3, 2, device="cuda")
    for f, m in [(-1, 1), (65536, 1), (1, 0), (1, 65536)]:
        with pytest.raises(RuntimeError):
            ext.krum_aggregate_slots(th, cp, n, f, m, 0, 0.0, 0.0, 1e-8, None, None, None, None, None)
    with pytest.raises(RuntimeError):
        ext.krum_aggregate_slots(th, cp, n, 1, 1, 2, 0.1, 0.0, 1e-8, None, None, None, None, None)   # adam without state
    with pytest.raises(RuntimeError):
        ext.krum_aggregate_slots(th, cp, n, 1, 1, 0, 0.0, 0.0, 1e-8, None, None, None, None,
                                 torch.ones(7, dtype=torch.uint8, device="cuda"))
    with pytest.raises(RuntimeError):
        ext.krum_aggregate_slots(th, cp, torch.ones(2, 2, device="cuda"), 1, 1, 0, 0.0, 0.0, 1e-8, None, None, None, None, None)
    with pytest.raises(ValueError):
        ops.fed_round_small(dict(to_cuda(make_state()), aggregation_rule="multi_krum", krum_m=0), 1)


def _kr(st, f=1, m=2):
    return dict(st, aggregation_rule="multi_krum", krum_f=f, krum_m=m)


SHAPES = [dict(), dict(kind="lr", hid=0), dict(din=2, hid=4), dict(kind="fnn", din=4, hid=8, dout=3), dict(C=37, M=4)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("wpp", [1, 2, 4])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_fused_matches_oracle_and_generic(shape, wpp, G):
    st = dict(_kr(make_state(**shape)), cluster=G, warps_per_pair=wpp)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 3)
    ref.fed_round_small(st, 3)
    torch.cuda.synchronize()
    assert torch.allclose(g["theta"].cpu(), st["theta"], rtol=1e-4, atol=1e-5), (g["theta"].cpu() - st["theta"]).abs().max()
    # one round on the kernel's own uploads: its aggregation equals K21 (and the oracle) applied to them
    C, M, P = st["X"].shape[1], *st["theta"].shape
    g["client_out"] = torch.zeros(C, M, P, device="cuda")
    theta0 = g["theta"].clone()
    ops.fed_round_small(g, 1)
    torch.cuda.synchronize()
    up = g["client_out"]
    sel = (up != 0).any(-1).float()
    k21 = theta0.clone()
    ops.krum_aggregate_slots_(k21, up, sel, 1, 2)
    want = theta0.cpu().clone()
    ref.krum_aggregate_slots_(want, up.cpu(), sel.cpu(), 1, 2)
    assert _same(g["theta"].cpu(), k21.cpu()) and _same(g["theta"].cpu(), want)


@pytest.mark.parametrize("f,m", [(0, 1), (3, 1), (1, 4), (2, 100)])
def test_fused_selection_parameters(f, m):
    st = dict(_kr(make_state(C=12), f, m), cluster=4)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    g["client_out"] = torch.zeros(C, M, P, device="cuda")
    theta0 = g["theta"].cpu().clone()
    ops.fed_round_small(g, 1)
    torch.cuda.synchronize()
    up = g["client_out"].cpu()
    want = theta0.clone()
    ref.krum_aggregate_slots_(want, up, (up != 0).any(-1).float(), f, m)
    assert _same(g["theta"].cpu(), want)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_fused_with_server_optimizer(kind):
    from test_server_opt import with_server_opt
    from test_gpu_server_opt import _compare
    st = with_server_opt(_kr(make_state()), kind)
    g = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(g, 3)
    ref.fed_round_small(st, 3)
    torch.cuda.synchronize()
    _compare(g, st)


def test_fused_is_bit_identical_across_runs_and_launch_splits():
    st = dict(_kr(make_state(C=12)), cluster=4)
    one, again, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    ops.fed_round_small(again, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    assert _same(one["theta"], again["theta"]) and _same(one["theta"], three["theta"])


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, aggregation_rule="multi_krum", krum_m=2)
    d.update(kw)
    return DriftSim(make_args(**d), device="cuda", sink=MetricsSink())


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
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert _same(a.bank.theta, b.bank.theta)


def test_fits_routes_and_cfg2_runs_fused():
    from feddrift_b200.experiments.configs import CONFIGS
    from feddrift_b200.ops import small_round
    # fnn 4-8-3 (P = 67, 8 warps): Multi-Krum needs C·(67 + 4·8 + 4) + 4 ≤ 8·33·67, so C ≤ 171
    assert small_round.fits("fnn", 4, 8, 3, 171, 2, 0, rule="multi_krum")
    assert not small_round.fits("fnn", 4, 8, 3, 172, 2, 0, rule="multi_krum")
    assert small_round.fits("fnn", 4, 8, 3, 172, 2, 0, robust=True)
    # lr 2-2 (P = 6, 16 warps): C·74 + 4 ≤ 3168, so C ≤ 42
    assert small_round.fits("lr", 2, 0, 2, 42, 2, 0, rule="multi_krum")
    assert not small_round.fits("lr", 2, 0, 2, 43, 2, 0, rule="multi_krum") and small_round.fits("lr", 2, 0, 2, 43, 2, 0)
    sim = _sim(client_num_in_total=100, sample_num=40, comm_round=2, total_train_iteration=2)
    sim.begin_time_step(0)
    assert sim._use_fused()
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    for name in ("cfg2_sea_fnn_100clients_feddrift", "cfg2k_sea_fnn_100clients_multikrum_feddrift"):
        cfg = dict(CONFIGS[name], aggregation_rule="multi_krum", comm_round=2, total_train_iteration=2)
        s = DriftSim(make_args(**cfg), device="cuda", sink=MetricsSink())
        s.begin_time_step(0)
        assert s._use_fused()
        n0 = small_round.LAUNCH_COUNT["fed_round_small"]
        s.run_rounds(2)
        assert small_round.LAUNCH_COUNT["fed_round_small"] > n0 and torch.isfinite(s.bank.theta).all()


def test_generic_executor_route():
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    sim = DriftSim(make_args(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                             concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                             total_train_iteration=2, epochs=2, aggregation_rule="multi_krum", krum_f=1, krum_m=2),
                   device="cuda", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    theta0 = sim.bank.theta.cpu().clone()
    sim.run_rounds(1)
    torch.cuda.synchronize()
    want = theta0.clone()
    mask = None if sim.defense_mask is None else sim.defense_mask.cpu()
    ref.krum_aggregate_slots_(want, sim.clients.params.cpu(), sim.clients.n.cpu(), 1, 2, mask)
    assert _same(sim.bank.theta.cpu(), want)


def test_byzantine_scenario_on_the_fused_kernel():
    from feddrift_b200.ops import small_round
    n0 = small_round.LAUNCH_COUNT["fed_round_small"]
    kr, sim = krum_honest_test_acc("cuda")
    assert sim._use_fused() and small_round.LAUNCH_COUNT["fed_round_small"] > n0
    mean, _ = honest_test_acc("mean", "cuda")
    assert kr >= KRUM_MIN and mean <= MEAN_MAX and np.isfinite(kr), (kr, mean)
