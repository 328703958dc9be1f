"""Coordinate-wise median and trimmed mean on the GPU: K19 (``robust_aggregate_slots``) bit for bit against the CPU oracle
(any client count, odd rows, padded banks, a ResNet-18-sized arena, every server optimizer), the fused round kernel's
aggregation phase (exactly against the oracle applied to the kernel's own uploads; multi-round runs against
``ref.fed_round_small``), launch modes, CUDA-graph replay, the generic executor's routes and the Byzantine scenario."""
import copy
import os

import numpy as np
import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.ops.server_opt import SlotServerOpt
from test_gpu_server_opt import CFGS, _compare, _table
from test_gpu_small_round import make_state, to_cuda
from test_robust_agg import BYZ, MEAN_MAX, ROBUST_MIN, _same, honest_test_acc
from test_server_opt import with_server_opt

pytestmark = pytest.mark.gpu
RULES = [("median", 0.1), ("trimmed_mean", 0.2)]


def _case(C, M, P, stride, seed=1, ties=False):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, stride, generator=g)
    up = torch.randn(C, M, P, generator=g)
    if ties:
        up = torch.tensor([-1.0, -0.0, 0.0, 0.5, 2.0])[torch.randint(0, 5, (C, M, P), generator=g)]
    n = (torch.rand(C, M, generator=g) * 4).floor()
    n[:, -1] = 0 if M > 1 else n[:, -1]    # the last slot has no participant (when there are several)
    return bank, up, n


@pytest.mark.parametrize("rule,beta", RULES)
@pytest.mark.parametrize("C,M,P,stride,ties", [
    (1, 2, 37, 37, False), (7, 3, 1001, 1001, False), (7, 3, 1003, 1024, True), (100, 2, 4096, 4096, False),
    (300, 2, 515, 520, True), (300, 1, 2048, 2048, False),
])
def test_k19_matches_reference_bit_for_bit(rule, beta, C, M, P, stride, ties):
    bank, up, n = _case(C, M, P, stride, ties=ties)
    up[0, 0, 5] = float("nan")
    want = bank.clone()
    cnt = ref.robust_aggregate_slots_(want[:, :P], up, n, rule, beta)
    gb = bank.cuda()
    got = ops.robust_aggregate_slots_(gb[:, :P], up.cuda(), n.cuda(), rule, beta)
    torch.cuda.synchronize()
    assert _same(gb.cpu(), want), (gb.cpu() != want).sum()
    assert torch.equal(got.cpu(), cnt)


def test_k19_resnet18_arena():
    P, C, M = 11_689_512, 32, 2
    g = torch.Generator().manual_seed(9)
    bank = torch.randn(M, P + 8, generator=g)
    up = torch.randn(C, M, P, generator=g)
    n = torch.ones(C, M)
    n[3, 1] = 0
    for rule, beta in RULES:
        want = bank.clone()
        ref.robust_aggregate_slots_(want[:, :P], up, n, rule, beta)
        gb = bank.cuda()
        ops.robust_aggregate_slots_(gb[:, :P], up.cuda(), n.cuda(), rule, beta)
        torch.cuda.synchronize()
        assert _same(gb.cpu(), want), rule


@pytest.mark.parametrize("kind", ["sgd", "adam", "adagrad", "yogi"])
@pytest.mark.parametrize("masked", [False, True])
def test_k19_with_server_optimizer(kind, masked):
    C, M, P = 9, 3, 1001
    bank, up, n = _case(C, M, P, P, seed=4)
    mask = (torch.arange(P) % 7 != 0) if masked else None
    hp = dict(lr=0.05, momentum=0.9 if kind == "sgd" else 0.0, eps=1e-3)
    for rule, beta in RULES:
        cpu_so = SlotServerOpt(kind, M, P, "cpu", mask=mask, **hp)
        gpu_so = SlotServerOpt(kind, M, P, "cuda", mask=mask, **hp)
        cpu, gpu = bank.clone(), bank.cuda()
        for _ in range(2):
            ops.cluster_aggregate_(cpu, up, n, cpu_so, (rule, beta))
            ops.cluster_aggregate_(gpu, up.cuda(), n.cuda(), gpu_so, (rule, beta))
        torch.cuda.synchronize()
        assert torch.equal(gpu_so.step.cpu(), cpu_so.step) and gpu_so.step.tolist() == [2, 2, 0]
        # the server step itself differs from the CPU law in the last bits (FMA contraction), as K1's epilogue does
        assert torch.allclose(gpu.cpu(), cpu, rtol=1e-4, atol=1e-5), (gpu.cpu() - cpu).abs().max()
        for a, b in zip(gpu_so.tensors(), cpu_so.tensors()):
            assert torch.allclose(a.cpu().float(), b.float(), rtol=1e-4, atol=1e-5)
        if mask is not None:   # entries outside the optimizer take the statistic itself
            avg = bank.clone()
            ref.robust_aggregate_slots_(avg, up, n, rule, beta)
            assert _same(gpu.cpu()[:2, ~mask], avg[:2, ~mask])


def test_binding_rejects_bad_input():
    ext = ops._ext.load()
    th, cp, n = torch.zeros(2, 8, device="cuda"), torch.zeros(3, 2, 8, device="cuda"), torch.ones(3, 2, device="cuda")
    with pytest.raises(RuntimeError):
        ext.robust_aggregate_slots(th, cp, n, 3, 0.1, 0, 0.0, 0.0, 1e-8, None, None, None, None)
    with pytest.raises(RuntimeError):
        ext.robust_aggregate_slots(th, cp, n, 2, 0.5, 0, 0.0, 0.0, 1e-8, None, None, None, None)
    with pytest.raises(RuntimeError):
        ext.robust_aggregate_slots(torch.zeros(3, 8, device="cuda"), cp, n, 1, 0.1, 0, 0.0, 0.0, 1e-8, None, None, None, None)
    with pytest.raises(RuntimeError):
        ext.robust_aggregate_slots(th, cp, n, 1, 0.1, 2, 0.1, 0.0, 1e-8, None, None, None, None)   # adam without state
    st = to_cuda(make_state())
    with pytest.raises(ValueError):
        ops.fed_round_small(dict(copy.deepcopy(st), aggregation_rule="krum"), 1)


def _one_round_against_own_uploads(st, rule, beta):
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].cpu().clone()
    st["client_out"] = torch.zeros(C, M, P, device="cuda")
    ops.fed_round_small(st, 1)
    torch.cuda.synchronize()
    up = st["client_out"].cpu()
    sel = (up != 0).any(-1)
    assert bool(sel.any())
    want = theta0.clone()
    ref.robust_aggregate_slots_(want, up, sel.float(), rule, beta)
    assert _same(st["theta"].cpu(), want), (st["theta"].cpu() - want).abs().max()


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("cfg", CFGS)
@pytest.mark.parametrize("rule,beta", RULES)
def test_fused_round_equals_oracle_rule_on_own_uploads(cfg, table, rule, beta):
    st = dict(make_state(**cfg), aggregation_rule=rule, trim_ratio=beta)
    if table:
        C = st["X"].shape[1]
        st["participation"] = _table(3, C, max(1, C // 3))
    st = to_cuda(st)
    for _ in range(2):
        _one_round_against_own_uploads(st, rule, beta)


def _multi_round(st_cpu, rounds=4):
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ops.fed_round_small(st_gpu, rounds)
    ref.fed_round_small(st_cpu, rounds)
    torch.cuda.synchronize()
    return st_gpu, st_cpu


@pytest.mark.parametrize("rule,beta", RULES)
@pytest.mark.parametrize("extra", [
    dict(recluster_hard=True, M=3), dict(defense="weak_dp", norm_bound=0.1, stddev=0.01),
    dict(compression="qsgd", quantize_level=4, quantize_bucket=8), dict(compression="eftopk", topk_ratio=0.3),
    dict(fedprox_mu=0.1),
])
def test_fused_multi_round_matches_reference(rule, beta, extra):
    extra = dict(extra)
    M = extra.pop("M", 4)
    st = dict(make_state(M=M), aggregation_rule=rule, trim_ratio=beta, **extra)
    g, c = _multi_round(st)
    assert torch.allclose(g["theta"].cpu(), c["theta"], rtol=1e-4, atol=1e-5), (g["theta"].cpu() - c["theta"]).abs().max()
    if extra.get("recluster_hard"):
        assert torch.equal(g["W"].cpu(), c["W"])


@pytest.mark.parametrize("kind", ["sgd", "adam", "adagrad", "yogi"])
def test_fused_multi_round_with_server_optimizer(kind):
    st = with_server_opt(dict(make_state(), aggregation_rule="median"), kind)
    st["participation"] = _table(3, 10, 4)
    g, c = _multi_round(st, 3)
    _compare(g, c)


def test_three_rounds_in_one_launch_equal_three_launches():
    st = dict(make_state(C=12), aggregation_rule="trimmed_mean", trim_ratio=0.25)
    st["participation"] = _table(3, 12, 6)
    one, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_step"):
        assert torch.equal(one[k], three[k]), k


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, aggregation_rule="median")
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
    assert torch.equal(a.bank.theta, b.bank.theta)


def test_cfg2_and_headline_run_on_the_fused_kernel():
    from feddrift_b200.experiments.configs import CONFIGS
    from feddrift_b200.ops import small_round
    from feddrift_b200.sim import make_args
    cfg = dict(CONFIGS["cfg2m_sea_fnn_100clients_median_feddrift"], comm_round=2, total_train_iteration=2)
    for kw in (cfg, dict(aggregation_rule="median", comm_round=2, total_train_iteration=2)):
        from feddrift_b200.sim import DriftSim
        from feddrift_b200.utils.metrics import MetricsSink
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.begin_time_step(0)
        assert sim._use_fused()
        n0 = small_round.LAUNCH_COUNT["fed_round_small"]
        sim.run_rounds(2)
        assert small_round.LAUNCH_COUNT["fed_round_small"] > n0
    # a shape whose ranking scratch does not fit goes to the generic executor, not to an error
    assert not small_round.fits("lr", 2, 0, 2, 200, 2, 0, robust=True) and small_round.fits("lr", 2, 0, 2, 200, 2, 0)


def _generic_rule(kw, env=None):
    """One round of time step 0 on the generic executor: θ must be the oracle rule applied to the raw arena, bit for bit."""
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        sim = DriftSim(make_args(aggregation_rule="median", **kw), device="cuda", sink=MetricsSink())
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        theta0 = sim.bank.theta.cpu().clone()
        sim.run_rounds(1)
        torch.cuda.synchronize()
        want = theta0.clone()
        ref.robust_aggregate_slots_(want, sim.clients.params.cpu(), sim.clients.n.cpu(), "median")
        assert _same(sim.bank.theta.cpu(), want)
        return sim
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_generic_per_pair_route():
    _generic_rule(dict(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                       concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                       total_train_iteration=2, epochs=2))


def test_generic_stacked_resnet18_route(monkeypatch):
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    _generic_rule(dict(model="resnet18", dataset="cifar10", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1",
                       concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=2,
                       total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05), {"FDB_STACKED": "force"})
    assert calls


def test_generic_lstm_route():
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    _generic_rule(dict(model="rnn", dataset="shakespeare", client_num_in_total=6, concept_num=2, concept_drift_algo="win-1",
                       concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16, comm_round=2,
                       total_train_iteration=2, epochs=2, lr=0.05, client_optimizer="sgd", report_client=0))
    assert fused.CALLS["bwd"] > n0


def test_byzantine_scenario_on_the_fused_kernel():
    from feddrift_b200.ops import small_round
    n0 = small_round.LAUNCH_COUNT["fed_round_small"]
    med, sim = honest_test_acc("median", "cuda")
    assert sim._use_fused() and small_round.LAUNCH_COUNT["fed_round_small"] > n0
    tm, _ = honest_test_acc("trimmed_mean", "cuda")
    mean, _ = honest_test_acc("mean", "cuda")
    assert med >= ROBUST_MIN and tm >= ROBUST_MIN, (med, tm, mean)
    assert mean <= MEAN_MAX, (med, tm, mean)
    assert BYZ == 3 and np.isfinite(med)
