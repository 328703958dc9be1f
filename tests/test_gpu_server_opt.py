"""Per-slot server optimizers on the GPU: the fused round kernel vs the CPU oracle, launch modes and CUDA-graph replay, the
extended K1 kernel vs the reference step, and the generic executor's routes.

Adam, Adagrad and Yogi normalise the pseudo-gradient: where it is tiny, a last-bit difference in the average (the kernel and
the oracle sum in different orders) can flip a step of size lr.  The comparisons therefore use τ = 1e-3, which bounds a step
by lr·|g|/τ."""
import copy

import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.ops.server_opt import SlotServerOpt
from feddrift_b200.sim.sampling import sample_clients
from test_gpu_small_round import make_state, to_cuda
from test_server_opt import HYPER, KINDS, with_server_opt

pytestmark = pytest.mark.gpu

CFGS = [dict(), dict(optimizer="sgd"), dict(kind="lr", hid=0), dict(din=2, hid=4), dict(B=32), dict(mode="time"),
        dict(mode="index", B=64), dict(C=37, M=4), dict(kind="fnn", din=4, hid=8, dout=3)]


def _table(rows, C, K):
    tab = torch.zeros(rows, C, dtype=torch.uint8)
    for r in range(rows):
        tab[r, torch.from_numpy(sample_clients(r, C, K))] = 1
    return tab


def _compare(st_gpu, st_cpu):
    # the adaptive kinds scale last-bit differences of the local models by up to lr/τ (= 50 here) per round
    atol = 2e-5 if st_cpu["server_opt"] == "sgd" else 1e-4
    assert torch.allclose(st_gpu["theta"].cpu(), st_cpu["theta"], rtol=2e-4, atol=atol), \
        (st_gpu["theta"].cpu() - st_cpu["theta"]).abs().max()
    assert torch.equal(st_gpu["server_step"].cpu(), st_cpu["server_step"])
    for k in ("server_s0", "server_s1"):
        if st_cpu[k] is not None:
            assert torch.allclose(st_gpu[k].cpu(), st_cpu[k], rtol=1e-3, atol=1e-6), (k, (st_gpu[k].cpu() - st_cpu[k]).abs().max())


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cfg", CFGS)
def test_fused_round_with_server_opt_matches_reference(cfg, kind, table):
    st_cpu = with_server_opt(make_state(**cfg), kind)
    C = st_cpu["X"].shape[1]
    if table:
        st_cpu["participation"] = _table(3, C, max(1, C // 3))
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu)
    assert int(st_cpu["server_step"].max()) > 0


def test_fused_round_with_server_opt_ifca_recluster():
    st_cpu = with_server_opt(make_state(M=3), "adam")
    st_cpu["recluster_hard"] = True
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 2)
    ops.fed_round_small(st_gpu, 2)
    torch.cuda.synchronize()
    Wg = st_gpu["W"][st_gpu["t_cur"]].cpu()
    assert torch.equal(Wg, st_cpu["W"][st_cpu["t_cur"]])
    _compare(st_gpu, st_cpu)


@pytest.mark.parametrize("kind", KINDS)
def test_three_rounds_in_one_launch_equal_three_launches(kind):
    st = with_server_opt(make_state(C=12), kind)
    st["participation"] = _table(3, 12, 4)
    one, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    for k in ("theta", "server_s0", "server_s1", "server_step", "opt_m", "opt_step"):
        if st[k] is not None:
            assert torch.equal(one[k], three[k]), k


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, server_optimizer="adam", server_lr=0.03, server_eps=1e-3)
    d.update(kw)
    return DriftSim(make_args(**d), device="cuda", sink=MetricsSink())


def test_round_graph_replay_matches_non_graph_path():
    def make():
        sim = _sim(client_num_per_round=3)
        for t in range(2):
            sim.run_time_step(t, rounds=4)
        sim.begin_time_step(2)
        sim.args.rounds_per_launch = 1
        sim.run_rounds(1)   # nonzero server state before the graph is built
        return sim

    a, b = make(), make()
    so = a.bank.server_opt
    before = [x.clone() for x in so.tensors()] + [a.bank.theta.clone()]
    ha, hb = a.make_host_round_inputs(), b.make_host_round_inputs()
    a._graph = (a._build_round_graph(ha), None)   # building the graph must not advance the experiment
    torch.cuda.synchronize()
    for x, y in zip(so.tensors() + [a.bank.theta], before):
        assert torch.equal(x, y)
    a._graph = None
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert torch.allclose(a.bank.theta, b.bank.theta, atol=1e-6)
    assert torch.equal(so.step, b.bank.server_opt.step)
    assert int(so.step.max()) == 5
    for x, y in zip(so.tensors(), b.bank.server_opt.tensors()):
        assert torch.allclose(x, y, rtol=1e-5, atol=1e-7)


def test_drift_sim_fused_path_uses_server_state():
    from feddrift_b200.ops import small_round
    sim = _sim(client_num_in_total=10)
    l0 = small_round.LAUNCH_COUNT["fed_round_small"]
    sim.run(end_iteration=2)
    assert small_round.LAUNCH_COUNT["fed_round_small"] > l0
    assert int(sim.bank.server_opt.step.max()) == 6 and bool((sim.bank.server_opt.s1 != 0).any())
    plain = _sim(client_num_in_total=10, server_optimizer="none")
    plain.run(end_iteration=2)
    assert not torch.allclose(sim.bank.theta, plain.bank.theta)


@pytest.mark.parametrize("P", [64, 37])
@pytest.mark.parametrize("kind", KINDS)
def test_cluster_aggregate_slots_matches_reference(kind, P):
    g = torch.Generator().manual_seed(11)
    C, M = 9, 4
    theta = torch.randn(M, P, generator=g)
    cp = theta[None] + 0.1 * torch.randn(C, M, P, generator=g)
    n = torch.rand(C, M, generator=g) + 0.1
    n[:, 1] = 0   # slot 1 does not aggregate
    mask = torch.rand(P, generator=g) > 0.2
    hp = HYPER[kind]
    mk = lambda dev: SlotServerOpt(kind, M, P, dev, lr=hp["server_lr"], momentum=hp.get("server_momentum", 0.0),  # noqa: E731
                                   eps=hp.get("server_eps", 1e-8), mask=mask)
    cpu, gpu = mk("cpu"), mk("cuda")
    for so in (cpu, gpu):   # different counters per slot: the bias correction is per slot
        so.step.copy_(torch.tensor([0, 7, 3, 12], dtype=torch.int32))
    th_c, th_g = theta.clone(), theta.cuda()
    for _ in range(3):
        ops.cluster_aggregate_(th_c, cp, n, cpu)
        tot = ops.cluster_aggregate_(th_g, cp.cuda(), n.cuda(), gpu)
    torch.cuda.synchronize()
    assert torch.allclose(tot.cpu(), n.sum(0), rtol=1e-6)
    assert gpu.step.tolist() == [3, 7, 6, 15] == cpu.step.tolist()
    assert torch.allclose(th_g.cpu(), th_c, rtol=1e-5, atol=1e-6), (th_g.cpu() - th_c).abs().max()
    assert torch.equal(th_g[1].cpu(), theta[1])
    for a, b in zip(gpu.tensors(), cpu.tensors()):
        assert torch.allclose(a.cpu().float(), b.float(), rtol=1e-4, atol=1e-7)
    # masked entries are the plain average and keep their state
    avg = theta.clone()
    ref.cluster_aggregate_(avg, cp, n)
    assert torch.allclose(th_g.cpu()[:, ~mask][[0, 2, 3]], avg[:, ~mask][[0, 2, 3]], rtol=1e-6, atol=1e-6)
    if gpu.s0 is not None:
        assert torch.all(gpu.s0[:, ~mask.cuda()] == 0)


def _generic(kw, env=None, rounds=2):
    """Run ``rounds`` single-round blocks of time step 0 on the generic executor and check each aggregation against the plain
    FedAvg of the same uploads: trainable entries are stepped, non-trainable ones (BatchNorm statistics) are the average."""
    import os
    from feddrift_b200.models import utils as mutils
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        sim = _sim(**kw)
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        so = sim.bank.server_opt
        wmask = mutils.weight_param_mask(sim.bank.spec)[: sim.bank.P].cuda()
        for _ in range(rounds):
            theta0, step0 = sim.bank.theta.clone(), so.step.clone()
            sim.run_rounds(1)
            torch.cuda.synchronize()
            avg = theta0.clone()
            ops.cluster_aggregate_(avg, sim.clients.params, sim.clients.n)   # plain FedAvg of this round's uploads
            trained = (sim.clients.n > 0).any(0)
            assert trained.any() and torch.equal(so.step - step0, trained.int())
            for m in range(sim.M):
                if not bool(trained[m]):
                    assert torch.equal(sim.bank.theta[m], theta0[m])
                    continue
                assert torch.allclose(sim.bank.theta[m, ~wmask], avg[m, ~wmask], rtol=1e-6, atol=1e-7)
                assert not torch.allclose(sim.bank.theta[m, wmask], avg[m, wmask])
        assert torch.isfinite(sim.bank.theta).all()
        return sim
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_generic_per_pair_graphs_apply_server_opt():
    sim = _generic(dict(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                        concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                        total_train_iteration=2, epochs=2))
    assert any(g.indexed and g.launches > 0 for g in sim.__dict__.get("_step_graphs", {}).values()), "per-pair graphs not used"


def test_generic_stacked_resnet_applies_server_opt_and_averages_bn_buffers(monkeypatch):
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    sim = _generic(dict(model="resnet18", dataset="cifar10", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1",
                        concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=2,
                        total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05), {"FDB_STACKED": "force"})
    assert calls
    assert sim.bank.server_opt.mask is not None and not bool(sim.bank.server_opt.mask.all())


def test_generic_lstm_applies_server_opt():
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    _generic(dict(model="rnn", dataset="shakespeare", client_num_in_total=6, concept_num=2, concept_drift_algo="win-1",
                  concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16, comm_round=2, total_train_iteration=2,
                  epochs=2, lr=0.05, client_optimizer="sgd", report_client=0))
    assert fused.CALLS["bwd"] > n0, "batched LSTM executor did not run"


def test_binding_rejects_bad_server_state():
    st = to_cuda(with_server_opt(make_state(), "adam"))
    bad = copy.deepcopy(st)
    bad["server_s1"] = None
    with pytest.raises(RuntimeError):
        ops.fed_round_small(bad, 1)
    bad = copy.deepcopy(st)
    bad["server_step"] = bad["server_step"].long()
    with pytest.raises(RuntimeError):
        ops.fed_round_small(bad, 1)
