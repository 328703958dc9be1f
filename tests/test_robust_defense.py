"""Robust aggregation (``--defense_type`` norm_diff_clipping / weak_dp) of the continual engines on the CPU: the round oracle
against a hand computation, the noise definition, composition with client sampling and a server optimizer, the device engine's
two routes, the raw-update hooks, BatchNorm entries, the façade's aggregation and the rejected configurations."""
import argparse
import copy

import pytest
import torch
from torch import nn

from feddrift_b200.core.robustness import make_defense
from feddrift_b200.models import utils as mutils
from feddrift_b200.ops import reference as ref
from feddrift_b200.parallel.arena import ModelBank
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state

DEFENSES = ["norm_diff_clipping", "weak_dp"]
STD = 0.01


def with_defense(st, defense, bound=0.1, stddev=STD):
    return dict(st, defense=defense, norm_bound=bound, stddev=stddev)


def _weights(st):
    """n_cm of every (client, slot) pair that trains at t_cur, as the oracle computes them."""
    C, M = st["X"].shape[1], st["theta"].shape[0]
    t, B = int(st["t_cur"]), int(st["batch_size"])
    nb = (st["nsamp"].to(torch.int64) + B - 1) // B
    active = (st["W"][t] != 0).any(dim=1)
    n = torch.zeros(C, M)
    for c in range(C):
        for m in range(M):
            if bool(active[m]):
                n[c, m] = ref._pair_plan(st, c, m, t, nb, B)[0]
    return n


@pytest.mark.parametrize("defense", DEFENSES)
def test_oracle_round_is_the_average_of_defended_uploads(defense):
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    a = with_defense(copy.deepcopy(st), defense)
    a["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(a, 1)
    plain = copy.deepcopy(st)
    plain["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(plain, 1)
    assert torch.equal(a["client_out"], plain["client_out"])   # the export holds the raw local models
    n = _weights(st)
    up = a["client_out"].clone()
    std = STD if defense == "weak_dp" else 0.0
    norms = ref.robust_clip_slots_(up, theta0, n, 0.1, None, std, ref.defense_seed(st["seed"], 0))
    assert bool((norms > 0.1).any())   # the bound is reached
    want = theta0.clone()
    for m in range(M):
        tot = n[:, m].double().sum()
        if tot > 0:
            want[m] = sum(up[c, m] * (float(n[c, m]) / float(tot)) for c in range(C) if n[c, m] > 0)
    assert torch.allclose(a["theta"], want, rtol=0, atol=1e-6), (a["theta"] - want).abs().max()
    assert torch.equal(a["theta"][3], theta0[3])   # slot 3 has no member at t_cur
    assert not torch.allclose(a["theta"], plain["theta"])
    for k in ("opt_m", "opt_step"):   # local training does not see the defense
        assert torch.equal(a[k], plain[k]), k


def test_unreached_bound_is_identical_to_none():
    st = make_state(C=8, S=40, epochs=2)
    a = with_defense(copy.deepcopy(st), "norm_diff_clipping", bound=1e30)
    plain = copy.deepcopy(st)
    ref.fed_round_small(a, 2)
    ref.fed_round_small(plain, 2)
    assert torch.equal(a["theta"], plain["theta"])
    s1, _ = _run(_sea(defense_type="norm_diff_clipping", norm_bound=1e30))
    s0, _ = _run(_sea())
    assert torch.equal(s1.bank.theta, s0.bank.theta)


def test_noise_is_gauss_hash_of_the_defense_seed():
    C, M, P = 3, 2, 37
    g = torch.Generator().manual_seed(0)
    theta = torch.randn(M, P + 5, generator=g)   # a padded bank row
    rows = theta[None, :, :P].repeat(C, 1, 1)   # zero update: the row becomes θ_m + stddev·z exactly
    n = torch.ones(C, M)
    n[1, 0] = 0
    seed = ref.defense_seed(1234, 5)
    ref.robust_clip_slots_(rows, theta, n, 1.0, None, 0.5, seed)
    z = ref.gauss_hash(seed, C * M, P).reshape(C, M, P)
    want = theta[None, :, :P] + 0.5 * z
    want[1, 0] = theta[0, :P]   # weight 0: untouched
    assert torch.equal(rows, want)
    assert torch.equal(ref.gauss_hash_rows(seed, [4, 1], P), ref.gauss_hash(seed, 5, P)[[4, 1]])
    assert len({ref.defense_seed(1234, r) for r in range(50)} | {ref.defense_seed(1235, 0)}) == 51


def test_composes_with_participation_and_server_adam():
    from test_server_opt import with_server_opt
    st = make_state(C=8, S=40, epochs=2)
    table = torch.zeros(2, 8, dtype=torch.bool)
    table[0, [0, 2, 5, 7]] = True
    table[1, [1, 3, 4, 5]] = True
    st["participation"] = table
    st = with_defense(st, "weak_dp")
    a = with_server_opt(copy.deepcopy(st), "adam")
    ref.fed_round_small(a, 1)
    plain = copy.deepcopy(st)   # the defended average without the server step
    ref.fed_round_small(plain, 1)
    want = with_server_opt(copy.deepcopy(st), "adam")
    active = torch.tensor([True, True, True, False])
    ref.server_opt_slots_(want["theta"], plain["theta"], active, "adam", want["server_s0"], want["server_s1"],
                          want["server_step"], want["server_lr"], 0.0, want["server_eps"])
    assert torch.equal(a["theta"], want["theta"])
    assert a["server_step"].tolist() == [1, 1, 1, 0]
    for c in (1, 3, 4, 6):   # non-participants did not train
        assert torch.equal(a["opt_step"][c], st["opt_step"][c])


def _sea(**kw):
    d = dict(client_num_in_total=8, comm_round=3, total_train_iteration=3, sample_num=40, epochs=2)
    d.update(kw)
    return make_args(**d)


def _run(args, end=None):
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    out = sim.run(end_iteration=end)
    return sim, out


@pytest.mark.parametrize("defense", DEFENSES)
def test_drift_sim_fused_and_generic_routes_agree(defense):
    args = _sea(defense_type=defense, norm_bound=0.01, stddev=STD)
    fused, out = _run(args, end=2)
    generic = DriftSim(copy.deepcopy(args), device="cpu", sink=MetricsSink())
    generic.algo.fused_ok = lambda: False
    generic.run(end_iteration=2)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    plain, _ = _run(_sea(), end=2)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, plain.bank.theta)
    assert all(h["test_acc"] == h["test_acc"] for h in out["history"])


def test_same_dummy_arg_gives_identical_runs():
    a, oa = _run(_sea(defense_type="weak_dp", norm_bound=0.01, dummy_arg=3))
    b, ob = _run(_sea(defense_type="weak_dp", norm_bound=0.01, dummy_arg=3))
    assert torch.equal(a.bank.theta, b.bank.theta) and oa["history"] == ob["history"]
    c, _ = _run(_sea(defense_type="weak_dp", norm_bound=0.01, dummy_arg=4))
    assert not torch.equal(a.bank.theta, c.bank.theta)


def _cnn_sim(**kw):
    d = dict(model="cnn", dataset="MNIST", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1", concept_drift_algo_arg="",
             change_points="A", sample_num=8, batch_size=8, comm_round=2, total_train_iteration=2, epochs=1, client_optimizer="sgd",
             lr=0.05)
    d.update(kw)
    sim = DriftSim(make_args(**d), device="cpu", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    return sim


@pytest.mark.parametrize("defense", DEFENSES)
def test_generic_cnn_round_aggregates_the_defended_arena(defense, monkeypatch):
    sim = _cnn_sim(defense_type=defense, norm_bound=0.01, stddev=STD)
    assert sim.spec is None
    theta0 = sim.bank.theta.clone()
    raw = []
    real = sim.defense.defend_slots_
    monkeypatch.setattr(sim.defense, "defend_slots_", lambda up, *a: (raw.append((up.clone(), a[1].clone())), real(up, *a))[1])
    sim.run_rounds(1)
    up, n = raw[0]   # the uploads as training left them
    std = STD if defense == "weak_dp" else 0.0
    norms = ref.robust_clip_slots_(up, theta0, n, 0.01, sim.defense_mask, std, ref.defense_seed(0 * 7919 + 13, 0))
    assert bool((norms > 0.01).any())
    sel = n > 0
    assert torch.allclose(sim.clients.params[sel], up[sel], rtol=0, atol=1e-6)
    want = theta0.clone()
    ref.cluster_aggregate_(want, up, n)
    assert torch.allclose(sim.bank.theta, want, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("algo", [("softcluster", "cfl_0.1_win-1"), ("clusterfl", "win-1")])
def test_raw_update_hooks_see_undefended_uploads(algo, monkeypatch):
    args = _sea(concept_drift_algo=algo[0], concept_drift_algo_arg=algo[1], concept_num=2, comm_round=3,
                defense_type="norm_diff_clipping", norm_bound=0.01)
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    sim.begin_time_step(0)
    seen = []
    if algo[0] == "clusterfl":
        sim.algo.split_round = 0
        real = sim.algo.on_client_updates
        monkeypatch.setattr(sim.algo, "on_client_updates", lambda t, p, n: (seen.append((p.clone(), n.clone())), real(t, p, n)))
    else:
        real = sim.algo.state.cluster_cfl
        monkeypatch.setattr(sim.algo.state, "cluster_cfl",
                            lambda t, r, bank, p, n: (seen.append((p.clone(), n.clone())), real(t, r, bank, p, n))[1])
    theta0 = sim.bank.theta.clone()
    sim.run_rounds(1)
    assert seen
    p, n = seen[0]
    sel = n > 0
    d = (p - theta0[None]).norm(dim=2)
    assert bool((d[sel] > 0.05).all())   # raw: well beyond the bound
    if algo[0] == "clusterfl":   # the aggregated arena is clipped (the split only moves uploads between slots)
        da = (sim.clients.params - sim.bank.theta[None]).norm(dim=2)
        assert torch.isfinite(da).all()


class _BnNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(1, 3, 3)
        self.bn = nn.BatchNorm2d(3)
        self.fc = nn.Linear(3 * 4 * 4, 2)

    def forward(self, x):
        return self.fc(torch.relu(self.bn(self.conv(x))).flatten(1))


@pytest.mark.parametrize("defense", DEFENSES)
def test_batchnorm_entries_pass_through(defense):
    bank = ModelBank(_BnNet(), 2, "cpu")
    P, M, C = bank.P, 2, 3
    wmask = mutils.weight_param_mask(bank.spec)[:P].bool()
    assert not bool(wmask.all())
    g = torch.Generator().manual_seed(1)
    bank.theta.copy_(torch.randn(M, P, generator=g))
    up = bank.theta[None] + torch.randn(C, M, P, generator=g)
    before = up.clone()
    d = make_defense(make_args(defense_type=defense, norm_bound=0.5, stddev=0.1))
    norms = d.defend_slots_(up, bank.theta, torch.ones(C, M), wmask, seed=9, rnd=2)
    assert torch.equal(up[..., ~wmask], before[..., ~wmask])
    want = (before - bank.theta[None])[..., wmask].norm(dim=2)
    assert torch.allclose(norms, want, rtol=1e-5)
    if defense == "norm_diff_clipping":
        assert torch.allclose((up - bank.theta[None])[..., wmask].norm(dim=2), torch.full((C, M), 0.5), rtol=1e-4)
    else:
        assert not torch.equal(up[..., wmask], before[..., wmask])


@pytest.mark.parametrize("defense", DEFENSES)
def test_facade_aggregation_defends_the_uploads(defense):
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    from feddrift_b200.fl.fedavg import FedAVGAggregator
    assert not FedAVGAggregator.defend_uploads   # fedavg_robust keeps its own single-model defense
    args = _sea(defense_type=defense, norm_bound=0.1, stddev=STD, dummy_arg=2, curr_train_iteration=1)
    M, C = 3, 5
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, C, "cpu", [model] * M, 2, args)
    P = agg.bank.P
    g = torch.Generator().manual_seed(3)
    agg.bank.theta.copy_(torch.randn(M, P, generator=g))
    std = STD if defense == "weak_dp" else 0.0
    seed = 2 * 7919 + 13 + 1000003 * 1
    for rnd in range(1, 3):
        theta0 = agg.bank.theta.clone()
        up = theta0[None] + 0.2 * torch.randn(C, M, P, generator=g)
        n = torch.randint(0, 3, (C, M), generator=g).float()
        n[:, -1] = 0
        agg.upload.copy_(up)
        agg.upload_n.copy_(n)
        agg._aggregate_models()
        want_up = up.clone()
        ref.robust_clip_slots_(want_up, theta0, n, 0.1, None, std, ref.defense_seed(seed, rnd))
        want = theta0.clone()
        ref.cluster_aggregate_(want, want_up, n)
        assert torch.equal(agg.bank.theta, want), rnd
        assert torch.equal(agg.bank.theta[-1], theta0[-1])
    plain = _BaseAggregator(None, None, None, None, None, None, None, C, "cpu", [model] * M, 2, _sea())
    assert plain.defense is None


@pytest.mark.parametrize("kw", [dict(defense_type="krum"), dict(defense_type="weak_dp", norm_bound=0.0),
                                dict(defense_type="norm_diff_clipping", norm_bound=-1.0),
                                dict(defense_type="norm_diff_clipping", norm_bound=float("inf")),
                                dict(defense_type="weak_dp", norm_bound=float("nan")), dict(defense_type="weak_dp", stddev=-0.1)])
def test_rejections(kw):
    with pytest.raises(ValueError):
        DriftSim(_sea(**kw), device="cpu", sink=MetricsSink())
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    with pytest.raises(ValueError):
        _BaseAggregator(None, None, None, None, None, None, None, 2, "cpu", [mutils.create_model("fnn", 2, 3)], 2, _sea(**kw))
    st = with_defense(make_state(C=8, S=20), kw["defense_type"], kw.get("norm_bound", 5.0), kw.get("stddev", 0.025))
    with pytest.raises(ValueError):
        ref.fed_round_small(st, 1)


def test_cli_flags():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.defense_type, a.norm_bound, a.stddev) == ("none", 5.0, 0.025)
    with pytest.raises(SystemExit):
        p.parse_args(["--defense_type", "krum"])
    from feddrift_b200.experiments.configs import CONFIGS
    assert CONFIGS["cfg2d_sea_fnn_100clients_weakdp_feddrift"]["defense_type"] == "weak_dp"
