"""Coordinate-wise median and trimmed-mean cluster aggregation (``--aggregation_rule``) of the continual engines on the CPU:
the oracle against an independent brute force, the trim count, permutation invariance, the round oracle's order of
operations, the device engine's two routes, checkpoint resume, the façade, the rejected configurations, the CLI and a
Byzantine scenario."""
import argparse
import copy
import itertools

import numpy as np
import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, checkpoint, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state
from test_robust_defense import _weights


def brute(theta, uploads, n, rule, beta):
    """Independent definition: a python sort of (value, client) per column, fp32 sum in rank order, one division."""
    out = theta.clone()
    C, M, P = uploads.shape
    for m in range(M):
        rows = [c for c in range(C) if float(n[c, m]) > 0]
        k = len(rows)
        if k == 0:
            continue
        b = (k - 1) // 2 if rule == "median" else int(np.floor(np.float32(beta) * np.float32(k)))
        for e in range(P):
            col = [np.float32(uploads[c, m, e].item()) for c in rows]
            if any(np.isnan(v) for v in col):
                out[m, e] = float("nan")
                continue
            order = sorted(range(k), key=lambda i: (float(col[i]) + 0.0, i))
            s = col[order[b]]
            for j in range(b + 1, k - b):
                s = np.float32(s + col[order[j]])
            out[m, e] = float(np.float32(s / np.float32(k - 2 * b)))
    return out


def _same(a, b):
    """Bit-identical, NaN included."""
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _arena(C, M=3, P=13, pad=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, P + pad, generator=g)
    return bank, torch.randn(C, M, P, generator=g), (torch.rand(C, M, generator=g) * 5).floor()


@pytest.mark.parametrize("rule,beta", [("median", 0.1), ("trimmed_mean", 0.0), ("trimmed_mean", 0.1), ("trimmed_mean", 0.25),
                                       ("trimmed_mean", 0.4999)])
@pytest.mark.parametrize("C", [1, 2, 7, 10])
def test_oracle_matches_brute_force(rule, beta, C):
    bank, up, n = _arena(C, pad=3)
    n[:, 1] = 0                       # a slot without participants keeps its model
    want = brute(bank, up, n, rule, beta)
    got = bank.clone()
    counts = ref.robust_aggregate_slots_(got[:, :13], up, n, rule, beta)
    assert _same(got, want)
    assert torch.equal(got[1], bank[1]) and torch.equal(got[:, 13:], bank[:, 13:])
    assert torch.equal(counts, (n > 0).sum(0).float())


@pytest.mark.parametrize("rule", ["median", "trimmed_mean"])
def test_ties_signed_zeros_infinities_and_nan(rule):
    C, M, P = 9, 1, 8
    vals = torch.tensor([0.0, -0.0, 1.0, -1.0, float("inf"), float("-inf"), 2.0, 2.0, 0.5])
    g = torch.Generator().manual_seed(5)
    up = torch.stack([vals[torch.randperm(C, generator=g)] for _ in range(P)], dim=1).reshape(C, M, P)
    up[:, 0, 0] = -0.0                # an all −0 column stays −0
    up[:, 0, 1] = torch.tensor([0.0, -0.0] * 4 + [0.0])
    up[3, 0, 2] = float("nan")        # a NaN column yields NaN
    up[:, 0, 3] = float("inf")
    n = torch.ones(C, M)
    theta = torch.zeros(M, P)
    want = brute(theta, up, n, rule, 0.3)
    got = theta.clone()
    ref.robust_aggregate_slots_(got, up, n, rule, 0.3)
    assert _same(got, want)
    assert got[0, 0].item() == 0.0 and torch.signbit(got[0, 0])
    assert torch.isnan(got[0, 2]) and got[0, 3].item() == float("inf")


def test_median_of_even_count_is_midpoint_and_n_one_is_identity():
    up = torch.tensor([[[1.0, 5.0]], [[3.0, -1.0]], [[10.0, 0.0]], [[2.0, 4.0]]])
    theta = torch.zeros(1, 2)
    ref.robust_aggregate_slots_(theta, up, torch.ones(4, 1), "median")
    assert theta.tolist() == [[2.5, 2.0]]
    one = torch.zeros(1, 2)
    ref.robust_aggregate_slots_(one, up[1:2], torch.ones(1, 1), "trimmed_mean", 0.49)
    assert torch.equal(one, up[1, 0:1])


def test_trim_count():
    assert ref.trim_count(0.1, 10) == 1 and ref.trim_count(0.0, 7) == 0 and ref.trim_count(0.49, 1) == 0
    assert ref.trim_count(0.3, 10) == 3       # fp32(0.3)·10 = 3 + 2⁻²³ rounds to 3 (ties to even)
    # β·n on an integer in decimal but not after fp32 rounding: 0.072·375 = 27, the fp32 product rounds below it
    assert ref.trim_count(0.072, 375) == 26
    # and fp32 keeps the integer where float64 drops below it: 0.35·180 = 63
    assert ref.trim_count(0.35, 180) == 63 and int(np.floor(0.35 * 180)) == 62
    for beta in (0.0, 0.1, 0.25, 0.4999):
        for n in (1, 2, 3, 10, 101):
            assert n - 2 * ref.trim_count(beta, n) >= 1


def test_aggregation_params():
    assert ref.aggregation_params("mean", 0.1) == ("mean", 0.1)
    assert ref.aggregation_params("median", 0) == ("median", 0.0)
    for rule, beta in [("krum", 0.1), ("Median", 0.1), ("mean", 0.5), ("median", -0.01), ("trimmed_mean", float("nan")),
                       ("mean", float("inf")), ("median", True), ("median", "x")]:
        with pytest.raises(ValueError):
            ref.aggregation_params(rule, beta)


@pytest.mark.parametrize("rule", ["median", "trimmed_mean"])
def test_permutation_invariance(rule):
    bank, up, n = _arena(6, M=2, P=31, seed=3)
    up[:, :, ::4] = up[0:1, :, ::4]   # columns full of ties
    base = bank.clone()
    ref.robust_aggregate_slots_(base, up, n, rule, 0.2)
    for perm in itertools.islice(itertools.permutations(range(6)), 0, 720, 97):
        got = bank.clone()
        ref.robust_aggregate_slots_(got, up[list(perm)], n[list(perm)], rule, 0.2)
        assert _same(got, base), perm


def test_trimmed_mean_beta_zero_is_the_unweighted_sorted_mean():
    bank, up, n = _arena(5, M=2, P=17, seed=7)
    n[:, :] = torch.tensor([1.0, 2.0, 3.0, 4.0, 50.0])[:, None]
    got = bank.clone()
    ref.robust_aggregate_slots_(got, up, n, "trimmed_mean", 0.0)
    srt = torch.sort(up, dim=0).values
    want = srt[0].clone()
    for j in range(1, 5):
        want = want + srt[j]
    assert _same(got, want / 5.0)
    weighted = bank.clone()
    ref.cluster_aggregate_(weighted, up, n)
    assert not torch.allclose(got, weighted, atol=1e-3)


def test_ops_dispatch_and_server_optimizer_on_cpu():
    from feddrift_b200.ops.server_opt import SlotServerOpt
    bank, up, n = _arena(7, M=3, P=11, seed=2)
    n[:, 2] = 0
    plain = bank.clone()
    assert torch.equal(ops.cluster_aggregate_(plain, up, n, None, ("median", 0.1)), (n > 0).sum(0).float())
    want = bank.clone()
    ref.robust_aggregate_slots_(want, up, n, "median")
    assert _same(plain, want)
    mean = bank.clone()
    ops.cluster_aggregate_(mean, up, n, None, ("mean", 0.1))
    w2 = bank.clone()
    ref.cluster_aggregate_(w2, up, n)
    assert torch.equal(mean, w2)
    so = SlotServerOpt("adam", 3, 11, "cpu", lr=0.1)
    th = bank.clone()
    ops.cluster_aggregate_(th, up, n, so, ("trimmed_mean", 0.2))
    avg = bank.clone()
    ref.robust_aggregate_slots_(avg, up, n, "trimmed_mean", 0.2)
    want = bank.clone()
    s0, s1, st = torch.zeros(3, 11), torch.zeros(3, 11), torch.zeros(3, dtype=torch.int32)
    ref.server_opt_slots_(want, avg, torch.tensor([True, True, False]), "adam", s0, s1, st, 0.1)
    assert torch.equal(th, want) and torch.equal(so.s0, s0) and so.step.tolist() == [1, 1, 0]


def _with_rule(st, rule, beta=0.2):
    return dict(st, aggregation_rule=rule, trim_ratio=beta)


@pytest.mark.parametrize("rule", ["median", "trimmed_mean"])
def test_oracle_round_applies_the_rule_after_compression_and_defense(rule):
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    n = _weights(st)
    # raw uploads (as compressed, undefended) from a mean run with the same compression: training does not see the rule
    kw = dict(compression="qsgd", quantize_level=4, quantize_bucket=8, defense="weak_dp", norm_bound=0.05, stddev=0.01)
    plain = dict(copy.deepcopy(st), **kw)
    plain["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(plain, 1)
    r = dict(_with_rule(copy.deepcopy(st), rule), **kw)
    r["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(r, 1)
    assert torch.equal(r["client_out"], plain["client_out"])   # client_out: compressed, not defended, rule-independent
    up = plain["client_out"].clone()
    ref.robust_clip_slots_(up, theta0, n, 0.05, None, 0.01, ref.defense_seed(st["seed"], 0))
    want = theta0.clone()
    ref.robust_aggregate_slots_(want, up, n, rule, 0.2)
    assert _same(r["theta"], want)
    # with a server optimizer: θ steps on θ − statistic
    so = dict(_with_rule(copy.deepcopy(st), rule), server_opt="adam", server_lr=0.05, server_s0=torch.zeros(M, P),
              server_s1=torch.zeros(M, P), server_step=torch.zeros(M, dtype=torch.int32))
    so["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(so, 1)
    avg = theta0.clone()
    ref.robust_aggregate_slots_(avg, so["client_out"], n, rule, 0.2)
    want = theta0.clone()
    s0, s1, stp = torch.zeros(M, P), torch.zeros(M, P), torch.zeros(M, dtype=torch.int32)
    ref.server_opt_slots_(want, avg, (n > 0).any(0), "adam", s0, s1, stp, 0.05)
    assert torch.equal(so["theta"], want) and torch.equal(so["server_step"], stp)


def _sea(**kw):
    d = dict(client_num_in_total=8, comm_round=3, total_train_iteration=3, sample_num=40, epochs=2)
    d.update(kw)
    return make_args(**d)


def _run(args, end=None, generic=False):
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    if generic:
        sim.algo.fused_ok = lambda: False
    out = sim.run(end_iteration=end)
    return sim, out


@pytest.mark.parametrize("rule", ["median", "trimmed_mean"])
def test_drift_sim_fused_and_generic_routes_agree(rule):
    args = _sea(aggregation_rule=rule, trim_ratio=0.2)
    fused, of = _run(args, end=2)
    generic, og = _run(copy.deepcopy(args), end=2, generic=True)
    assert fused.agg_rule == (rule, 0.2)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    plain, _ = _run(_sea(), end=2)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, plain.bank.theta)
    assert _run(_sea(aggregation_rule="mean", trim_ratio=0.3), end=2)[0].bank.theta.equal(plain.bank.theta)


def test_generic_cnn_round_takes_the_rule_of_the_raw_arena(monkeypatch):
    calls = []
    real = ops.cluster_aggregate_

    def wrapped(theta, cp, n, server_opt=None, rule=None):
        calls.append((theta.clone(), cp.clone(), n.clone(), rule))
        return real(theta, cp, n, server_opt, rule)
    monkeypatch.setattr(ops, "cluster_aggregate_", wrapped)
    sim = DriftSim(make_args(model="cnn", dataset="MNIST", client_num_in_total=5, concept_num=2, concept_drift_algo="win-1",
                             concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=1,
                             total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05, aggregation_rule="median"),
                   device="cpu", sink=MetricsSink())
    assert sim.spec is None
    sim.begin_time_step(0)
    sim.run_rounds(1)
    theta0, cp, n, rule = calls[0]
    assert rule == ("median", 0.1)
    want = theta0.clone()
    ref.robust_aggregate_slots_(want, cp, n, "median")
    assert _same(sim.bank.theta, want)


def test_checkpoint_resume_with_median(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, aggregation_rule="trimmed_mean", trim_ratio=0.25)
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    full.run()
    part = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    part.run(0, 2)
    resumed = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    nxt = checkpoint.resume(resumed, checkpoint.latest(str(tmp_path)))
    assert nxt == 2
    resumed.run(nxt)
    assert torch.equal(resumed.bank.theta, full.bank.theta)


def test_facade_aggregator_uses_the_rule():
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    from feddrift_b200.models import utils as mutils
    M, W = 2, 5
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, W, "cpu", [model] * M, 2,
                          _sea(aggregation_rule="median", client_num_in_total=W))
    P = agg.bank.P
    g = torch.Generator().manual_seed(3)
    agg.bank.theta.copy_(torch.randn(M, P, generator=g))
    theta0 = agg.bank.theta.clone()
    raw = theta0[None] + torch.randn(W, M, P, generator=g)
    for w in range(W):
        sds = {m: ({k: v.clone() for k, v in mutils.unflatten_to_state_dict(raw[w, m], agg.bank.spec).items()},
                   0 if (m == 1 and w == 0) else 3 + w) for m in range(M)}
        agg.add_local_trained_result(w, sds)
    assert agg.check_whether_all_receive()
    agg._aggregate_models()
    n = agg.upload_n.clone()
    want = theta0.clone()
    ref.robust_aggregate_slots_(want, raw, n, "median")
    assert _same(agg.bank.theta, want)


def test_facade_inproc_matches_the_engine():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args, run_device, run_facade
    from feddrift_b200.utils.metrics import set_sink
    base = ["--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60", "--aggregation_rule", "median"]
    p = add_args(argparse.ArgumentParser())
    sf, se, sm = MetricsSink(), MetricsSink(), MetricsSink()
    f = run_facade(p.parse_args(["--engine", "facade"] + base), set_sink(sf))
    e = run_device(p.parse_args(["--engine", "device"] + base), set_sink(se))
    run_facade(p.parse_args(["--engine", "facade", "--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60"]),
               set_sink(sm))
    assert len(f["history"]) == 2
    assert np.allclose(sf.series("Test/Acc"), se.series("Test/Acc"), atol=0.02)
    assert sf.series("Train/Loss") != sm.series("Train/Loss")


@pytest.mark.parametrize("kw", [dict(aggregation_rule="krum"), dict(aggregation_rule="median", trim_ratio=0.5),
                                dict(aggregation_rule="mean", trim_ratio=-0.1),
                                dict(aggregation_rule="trimmed_mean", trim_ratio=float("nan"))])
def test_rejections(kw):
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    from feddrift_b200.models import utils as mutils
    with pytest.raises(ValueError):
        DriftSim(_sea(**kw), device="cpu", sink=MetricsSink())
    with pytest.raises(ValueError):
        _BaseAggregator(None, None, None, None, None, None, None, 2, "cpu", [mutils.create_model("fnn", 2, 3)], 2, _sea(**kw))
    with pytest.raises(ValueError):
        ref.fed_round_small(dict(make_state(C=8, S=20), **kw), 1)


def test_multi_gpu_is_rejected():
    sim = DriftSim(_sea(aggregation_rule="median"), device="cpu", sink=MetricsSink())
    from feddrift_b200.parallel.symm import attach_multi_gpu
    with pytest.raises(ValueError, match="aggregation_rule"):
        attach_multi_gpu(sim, 2, 0)
    sim.shard_clients = True
    with pytest.raises(ValueError, match="aggregation_rule"):
        sim.run_time_step(0)
    sim2 = DriftSim(_sea(aggregation_rule="median"), device="cpu", sink=MetricsSink())
    sim2.multi = {"world": 2}
    with pytest.raises(ValueError, match="aggregation_rule"):
        sim2.run_time_step(0)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.aggregation_rule, a.trim_ratio) == ("mean", 0.1)
    assert (make_args().aggregation_rule, make_args().trim_ratio) == ("mean", 0.1)
    a = p.parse_args(["--aggregation_rule", "trimmed_mean", "--trim_ratio", "0.3"])
    assert (a.aggregation_rule, a.trim_ratio) == ("trimmed_mean", 0.3)
    with pytest.raises(SystemExit):
        p.parse_args(["--aggregation_rule", "krum"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2m_sea_fnn_100clients_median_feddrift"]
    assert cfg["aggregation_rule"] == "median" and cfg["client_num_in_total"] == 100


# ----------------------------------------------------------------------------- Byzantine scenario
BYZ = 3   # clients 0..2 flip their labels and scale their features by 100
BYZ_KW = dict(dataset="sea", client_num_in_total=10, client_num_per_round=10, concept_drift_algo="win-1", concept_drift_algo_arg="",
              client_optimizer="sgd", lr=0.5, comm_round=20, total_train_iteration=3, sample_num=100, epochs=2,
              change_points="A")
# thresholds fixed from the CPU run (honest clients' mean Test/Acc after the last round: median ≈ 0.71, mean 0.60, the
# majority class: the attackers' updates swamp the average)
ROBUST_MIN, MEAN_MAX = 0.67, 0.62


def byzantine_data():
    from feddrift_b200.sim.engine import generate_drift_data
    a = make_args(**BYZ_KW)
    data = generate_drift_data(a.dataset, a.total_train_iteration, a.client_num_in_total, a.sample_num, a.noise_prob,
                               a.time_stretch, a.change_points, bool(a.drift_together), seed=0)
    data.X[:, :BYZ] *= 100.0
    data.Y[:, :BYZ] = 1 - data.Y[:, :BYZ]
    return data


def honest_test_acc(rule, device="cpu", beta=0.3):
    sim = DriftSim(make_args(aggregation_rule=rule, trim_ratio=beta, **BYZ_KW), data=byzantine_data(), device=device,
                   sink=MetricsSink())
    sim.run()
    accs = [sim.sink.series(f"Test/Acc-CL-{c}")[-1] for c in range(BYZ, 10)]
    return float(np.mean(accs)), sim


def test_byzantine_clients_median_and_trimmed_mean_hold():
    med, _ = honest_test_acc("median")
    tm, _ = honest_test_acc("trimmed_mean")
    mean, _ = honest_test_acc("mean")
    assert med >= ROBUST_MIN and tm >= ROBUST_MIN, (med, tm, mean)
    assert mean <= MEAN_MAX, (med, tm, mean)
