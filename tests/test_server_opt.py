"""Per-slot server optimizers (``--server_optimizer``) of the continual engines on the CPU: the round oracle's composition,
equivalences with plain FedAvg, state resets, checkpoint resume, the BatchNorm mask of the generic aggregation, the façade's
aggregation and the rejected configurations."""
import copy

import pytest
import torch
from torch import nn

from feddrift_b200 import ops
from feddrift_b200.models import utils as mutils
from feddrift_b200.ops import reference as ref
from feddrift_b200.ops.server_opt import SlotServerOpt, make_server_opt
from feddrift_b200.parallel.arena import ModelBank
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state

KINDS = ["sgd", "adam", "adagrad", "yogi"]
HYPER = {"sgd": dict(server_lr=1.0, server_momentum=0.9), "adam": dict(server_lr=0.05, server_eps=1e-3),
         "adagrad": dict(server_lr=0.05, server_eps=1e-3), "yogi": dict(server_lr=0.05, server_eps=1e-3)}


def with_server_opt(st, kind, **over):
    """``st`` plus fresh per-slot state for ``kind`` (the keys ``reference.fed_round_small`` documents)."""
    M, P = st["theta"].shape
    hp = dict(HYPER[kind], **over)
    so = SlotServerOpt(kind, M, P, "cpu", lr=hp["server_lr"], momentum=hp.get("server_momentum", 0.0),
                       eps=hp.get("server_eps", 1e-8))
    st = dict(st, server_opt=kind, server_s0=so.s0, server_s1=so.s1, server_step=so.step, **hp)
    return st


@pytest.mark.parametrize("empty_cluster", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_round_is_plain_round_plus_slot_step(kind, empty_cluster):
    st = with_server_opt(make_state(C=8, S=40, epochs=2), kind)
    # nonzero starting state and counters, different per slot
    g = torch.Generator().manual_seed(7)
    if st["server_s0"] is not None:
        st["server_s0"].copy_(torch.rand(st["server_s0"].shape, generator=g) * 0.01)
    if st["server_s1"] is not None:
        st["server_s1"].copy_(torch.rand(st["server_s1"].shape, generator=g) * 0.01)
    st["server_step"].copy_(torch.tensor([3, 0, 5, 2], dtype=torch.int32))
    if empty_cluster:   # client 5 is cluster 2's only member at t_cur (make_state's plan): a table without it empties slot 2
        table = torch.ones(1, 8, dtype=torch.bool)
        table[0, 5] = False
        st["participation"] = table
    a = copy.deepcopy(st)
    ref.fed_round_small(a, 1)
    plain = copy.deepcopy(st)
    for k in ("server_opt", "server_s0", "server_s1", "server_step"):
        plain.pop(k)
    ref.fed_round_small(plain, 1)
    want = copy.deepcopy(st)
    active = torch.tensor([True, True, not empty_cluster, False])   # slot 3 has no member at t_cur
    ref.server_opt_slots_(want["theta"], plain["theta"], active, kind, want["server_s0"], want["server_s1"], want["server_step"],
                          st["server_lr"], st.get("server_momentum", 0.0), st.get("server_eps", 1e-8))
    for k in ("theta", "server_s0", "server_s1", "server_step"):
        if st[k] is not None:
            assert torch.equal(a[k], want[k]), k
    for k in ("opt_m", "opt_step"):   # local training does not see the server optimizer
        assert torch.equal(a[k], plain[k]), k
    assert a["server_step"].tolist() == [4, 1, 5 if empty_cluster else 6, 2]
    for m in [3] + ([2] if empty_cluster else []):   # slots that did not aggregate: θ, state and counter bit-identical
        for k in ("theta", "server_s0", "server_s1"):
            if st[k] is not None:
                assert torch.equal(a[k][m], st[k][m]), (k, m)
    assert not torch.equal(a["theta"][0], plain["theta"][0])


def _sea(**kw):
    d = dict(client_num_in_total=8, comm_round=3, total_train_iteration=3, sample_num=40, epochs=2)
    d.update(kw)
    return make_args(**d)


def _run(args, end=None):
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    out = sim.run(end_iteration=end)
    return sim, out


def test_none_is_bit_identical_to_default():
    a, oa = _run(_sea())
    b, ob = _run(_sea(server_optimizer="none", server_lr=0.3))
    assert b.bank.server_opt is None
    assert torch.equal(a.bank.theta, b.bank.theta)
    assert oa["history"] == ob["history"]


def test_sgd_lr1_without_momentum_is_fedavg():
    a, _ = _run(_sea())
    b, _ = _run(_sea(server_optimizer="sgd", server_lr=1.0, server_momentum=0.0))
    assert b.bank.server_opt is not None and int(b.bank.server_opt.step.max()) > 0
    assert torch.allclose(a.bank.theta, b.bank.theta, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("algo", [("softcluster", "H_A_C_1_10_0"), ("softclusterwin-1", "hard-r")])
def test_drift_sim_feddrift_and_ifca_with_adam(algo):
    args = _sea(concept_drift_algo=algo[0], concept_drift_algo_arg=algo[1], server_optimizer="adam", server_lr=0.03,
                server_eps=1e-3)
    sim, out = _run(args)
    plain, _ = _run(_sea(concept_drift_algo=algo[0], concept_drift_algo_arg=algo[1]))
    assert len(out["history"]) == 3 and all(h["test_acc"] == h["test_acc"] for h in out["history"])
    so = sim.bank.server_opt
    assert torch.isfinite(sim.bank.theta).all() and int(so.step.max()) == 3   # counters restart every time step
    assert not torch.allclose(sim.bank.theta, plain.bank.theta)


def test_state_resets_at_every_time_step():
    sim = DriftSim(_sea(server_optimizer="yogi", server_lr=0.05, server_eps=1e-3), device="cpu", sink=MetricsSink())
    sim.run_time_step(0)
    so = sim.bank.server_opt
    assert int(so.step[0]) == 3 and not torch.all(so.s0 == 0) and not torch.all(so.s1 == 1e-6)
    sim.begin_time_step(1)
    assert torch.all(so.step == 0) and torch.all(so.s0 == 0) and torch.all(so.s1 == 1e-6)


def test_bank_reinit_and_copy_reset_the_destination_slot():
    bank = ModelBank(mutils.create_model("fnn", 2, 3), 3, "cpu")
    bank.server_opt = SlotServerOpt("adam", 3, bank.P, "cpu", lr=0.1)
    so = bank.server_opt
    so.s0.fill_(0.5); so.s1.fill_(0.25); so.step.fill_(4)
    bank.copy(1, 0)
    assert torch.all(so.s0[1] == 0) and torch.all(so.s1[1] == 0) and int(so.step[1]) == 0
    assert torch.all(so.s0[0] == 0.5) and int(so.step[0]) == 4 and int(so.step[2]) == 4
    bank.reinit(2)
    assert torch.all(so.s0[2] == 0) and int(so.step[2]) == 0 and int(so.step[0]) == 4
    bank.copy(0, 0)   # a self-copy overwrites nothing
    assert int(so.step[0]) == 4


def test_clusterfl_split_resets_the_new_slot(monkeypatch):
    sim = DriftSim(_sea(concept_drift_algo="clusterfl", concept_drift_algo_arg="win-1", concept_num=2, comm_round=5,
                        server_optimizer="adam", server_lr=0.03, server_eps=1e-3), device="cpu", sink=MetricsSink())
    sim.algo.split_round = 2
    resets = []
    real = sim.bank.server_opt.reset
    monkeypatch.setattr(sim.bank.server_opt, "reset", lambda m=None: (resets.append(m), real(m)))
    sim.run_time_step(0)
    assert sim.algo.split_done and 1 in resets
    assert int(sim.bank.server_opt.step[0]) == 5 and 0 < int(sim.bank.server_opt.step[1]) < 5


def test_checkpoint_resume_matches_uninterrupted_run(tmp_path):
    kw = dict(server_optimizer="adam", server_lr=0.03, server_eps=1e-3)
    full, _ = _run(_sea(checkpoint_dir=str(tmp_path / "a"), **kw))
    from feddrift_b200.sim import checkpoint as ckpt
    first = DriftSim(_sea(checkpoint_dir=str(tmp_path / "b"), **kw), device="cpu", sink=MetricsSink())
    first.run(end_iteration=2)
    resumed = DriftSim(_sea(checkpoint_dir=str(tmp_path / "b"), **kw), device="cpu", sink=MetricsSink())
    start = ckpt.resume(resumed, ckpt.latest(str(tmp_path / "b")))
    assert start == 2
    resumed.run(start_iteration=start)
    assert torch.equal(resumed.bank.theta, full.bank.theta)


class _BnNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(1, 3, 3)
        self.bn = nn.BatchNorm2d(3)
        self.fc = nn.Linear(3 * 4 * 4, 2)

    def forward(self, x):
        return self.fc(torch.relu(self.bn(self.conv(x))).flatten(1))


@pytest.mark.parametrize("kind", KINDS)
def test_generic_aggregation_masks_batchnorm_buffers(kind):
    bank = ModelBank(_BnNet(), 3, "cpu")
    P, M, C = bank.P, 3, 5
    wmask = mutils.weight_param_mask(bank.spec)[:P]
    assert not bool(wmask.all())
    so = make_server_opt(make_args(server_optimizer=kind, **HYPER[kind]), M, P, "cpu", mutils.weight_param_mask(bank.spec))
    assert so.mask is not None and torch.equal(so.mask, wmask)
    g = torch.Generator().manual_seed(1)
    bank.theta.copy_(torch.randn(M, P, generator=g))
    cp = bank.theta[None] + 0.1 * torch.randn(C, M, P, generator=g)
    n = torch.rand(C, M, generator=g) + 0.5
    n[:, 2] = 0   # slot 2 has no upload: untouched
    theta0 = bank.theta.clone()
    avg = bank.theta.clone()
    ref.cluster_aggregate_(avg, cp, n)
    want = bank.theta.clone()
    for m in range(2):   # FedOpt on the trainable entries only, as fl/standalone.py's FedOptTrainer does
        w = want[m, wmask]
        ref.server_opt_step_(w, avg[m, wmask], {}, kind, HYPER[kind]["server_lr"],
                             **({"momentum": 0.9} if kind == "sgd" else {"eps": 1e-3}))
        want[m, wmask] = w
    ops.cluster_aggregate_(bank.theta, cp, n, so)
    assert torch.equal(bank.theta[:2, ~wmask], avg[:2, ~wmask])   # BN statistics: the plain average
    assert torch.equal(bank.theta[2], theta0[2])
    assert torch.allclose(bank.theta[:2, wmask], want[:2, wmask], rtol=1e-5, atol=1e-6)
    assert so.step.tolist() == [1, 1, 0]


def test_generic_executor_applies_server_opt():
    args = _sea(server_optimizer="adam", server_lr=0.03, server_eps=1e-3)
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    fused = DriftSim(copy.deepcopy(args), device="cpu", sink=MetricsSink())
    for s in (sim, fused):
        s.run(end_iteration=2)
    assert torch.equal(sim.bank.server_opt.step, fused.bank.server_opt.step)
    assert torch.allclose(sim.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)   # same semantics as the oracle


@pytest.mark.parametrize("kind", KINDS)
def test_facade_and_drift_sim_apply_the_same_server_step(kind):
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    args = _sea(server_optimizer=kind, **HYPER[kind])
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    M, P, C = sim.M, sim.bank.P, sim.C
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, C, "cpu", [model] * M, 2, args)
    agg.bank.theta.copy_(sim.bank.theta)
    g = torch.Generator().manual_seed(3)
    for rnd in range(3):
        up = sim.bank.theta[None] + 0.05 * torch.randn(C, M, P, generator=g)
        n = torch.randint(0, 3, (C, M), generator=g).float()
        n[:, -1] = 0
        agg.upload.copy_(up)
        agg.upload_n.copy_(n)
        agg._aggregate_models()
        sim.clients.params.copy_(up)
        sim.clients.n.copy_(n)
        ops.cluster_aggregate_(sim.bank.theta, sim.clients.params, sim.clients.n, sim.bank.server_opt)   # sim/generic.py's call
        assert torch.equal(agg.bank.theta, sim.bank.theta), rnd
    assert torch.equal(agg.bank.server_opt.step, sim.bank.server_opt.step)
    assert int(sim.bank.server_opt.step[-1]) == 0


def test_rejections():
    with pytest.raises(ValueError):
        DriftSim(_sea(server_optimizer="rmsprop"), device="cpu", sink=MetricsSink())
    sim = DriftSim(_sea(server_optimizer="adam"), device="cpu", sink=MetricsSink())
    from feddrift_b200.parallel.symm import attach_multi_gpu
    with pytest.raises(ValueError):
        attach_multi_gpu(sim, 2, 0)
    sim.shard_clients = True
    with pytest.raises(ValueError):
        sim.run_time_step(0)
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    import argparse
    with pytest.raises(SystemExit):
        add_args(argparse.ArgumentParser()).parse_args(["--server_optimizer", "rmsprop"])
