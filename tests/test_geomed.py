"""Geometric-median cluster aggregation (``--aggregation_rule geometric_median``) of the continual engines on the CPU: the
oracle against an independent float64 Weiszfeld, optimality, rotation equivariance, breakdown, the edge cases, the server
optimizer, the device engine's two routes, checkpoint resume, the façade, the rejected configurations, the CLI and the
Byzantine scenario."""
import argparse
import copy

import numpy as np
import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, checkpoint, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state
from test_robust_agg import BYZ, MEAN_MAX, _same, honest_test_acc
from test_robust_defense import _weights


def weiszfeld(theta, uploads, n, iters=4, nu=1e-6, mask=None):
    """Independent definition in numpy: start at the coordinate-wise median (np.median of the fp32 column), then float64
    smoothed Weiszfeld steps; rows whose weight is 0 are left out; a NaN distance makes the slot NaN; W = 0 keeps v."""
    out = theta.double().numpy().copy()
    X = uploads.numpy()
    C, M, P = X.shape
    keep = np.ones(P, bool) if mask is None else mask.numpy().astype(bool)
    for m in range(M):
        rows = [c for c in range(C) if float(n[c, m]) > 0]
        if not rows:
            continue
        x = X[rows, m, :]                                  # float32
        v = np.median(x, axis=0).astype(np.float64)
        if len(rows) > 2:
            xd = x.astype(np.float64)
            for _ in range(iters):
                with np.errstate(invalid="ignore"):
                    d = np.sqrt((((xd - v) ** 2) * keep).sum(1))
                if np.isnan(d).any():
                    v = np.full(P, np.nan)
                    break
                w = 1.0 / np.maximum(nu, d)
                if w.sum() == 0:
                    break
                on = w != 0
                v = (w[on, None] * xd[on]).sum(0) / w[on].sum()
        out[m, :P] = v
    return torch.from_numpy(out)


def _arena(C, M=3, P=13, pad=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, P + pad, generator=g)
    return bank, torch.randn(C, M, P, generator=g), (torch.rand(C, M, generator=g) * 5).floor() + (torch.arange(C) % 2)[:, None]


def _close(a, b, rtol=1e-5, atol=1e-6):
    return torch.allclose(a.double(), b.double(), rtol=rtol, atol=atol, equal_nan=True)


@pytest.mark.parametrize("C", [1, 2, 3, 7, 10])
@pytest.mark.parametrize("masked", [False, True])
def test_oracle_matches_numpy_weiszfeld(C, masked):
    bank, up, n = _arena(C, pad=3, seed=C)
    n[:, 1] = 0                                          # a slot without participants keeps its model
    mask = (torch.arange(13) % 5 != 2) if masked else None
    if masked:
        up[:, :, ~mask] *= 100.0                         # BatchNorm-like statistics: aggregated, out of the distance
    want = weiszfeld(bank, up, n, mask=mask)
    got = bank.clone()
    counts = ref.geomed_aggregate_slots_(got[:, :13], up, n, 4, 1e-6, mask)
    assert _close(got, want), (got.double() - want).abs().max()
    assert torch.equal(got[1], bank[1]) and torch.equal(got[:, 13:], bank[:, 13:])
    assert torch.equal(counts, (n > 0).sum(0).float())
    if masked and C > 2:   # the masked entries do steer nothing: scaling them again leaves the trainable entries unchanged
        up2 = up.clone()
        up2[:, :, ~mask] *= 3.0
        got2 = bank.clone()
        ref.geomed_aggregate_slots_(got2[:, :13], up2, n, 4, 1e-6, mask)
        assert torch.equal(got2[:, :13][:, mask], got[:, :13][:, mask])


def _objective(v, x):
    return float(np.linalg.norm(x - v[None], axis=1).sum())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_optimality_against_scipy(seed):
    from scipy.optimize import minimize
    g = torch.Generator().manual_seed(seed)
    k, P = 9, 4
    up = torch.randn(k, 1, P, generator=g) * torch.tensor([1.0, 3.0, 0.5, 2.0])
    theta = torch.zeros(1, P)
    ref.geomed_aggregate_slots_(theta, up, torch.ones(k, 1), 100, 1e-9)
    x = up[:, 0].double().numpy()
    v = theta[0].double().numpy()
    best = minimize(lambda z: _objective(z, x), x.mean(0), method="Nelder-Mead",
                    options=dict(xatol=1e-10, fatol=1e-12, maxiter=20000, maxfev=40000))
    f = _objective(v, x)
    assert f <= best.fun * (1 + 1e-5), (f, best.fun)
    med = theta.clone()
    ref.robust_aggregate_slots_(med, up, torch.ones(k, 1), "median")
    assert f <= _objective(x.mean(0), x) and f <= _objective(med[0].double().numpy(), x)


def test_rotation_equivariance():
    g = torch.Generator().manual_seed(4)
    k, P = 8, 6
    up = torch.randn(k, 1, P, generator=g, dtype=torch.float64)
    Q, _ = torch.linalg.qr(torch.randn(P, P, generator=g, dtype=torch.float64))
    a, b = torch.zeros(1, P), torch.zeros(1, P)
    ref.geomed_aggregate_slots_(a, up.float(), torch.ones(k, 1), 100, 1e-9)
    ref.geomed_aggregate_slots_(b, (up @ Q.T).float(), torch.ones(k, 1), 100, 1e-9)
    assert torch.allclose(b.double(), a.double() @ Q.T, atol=1e-4), (b.double() - a.double() @ Q.T).abs().max()
    # the coordinate-wise median is not equivariant
    ma, mb = torch.zeros(1, P), torch.zeros(1, P)
    ref.robust_aggregate_slots_(ma, up.float(), torch.ones(k, 1), "median")
    ref.robust_aggregate_slots_(mb, (up @ Q.T).float(), torch.ones(k, 1), "median")
    assert not torch.allclose(mb.double(), ma.double() @ Q.T, atol=1e-2)


def test_breakdown_four_of_ten_far_outliers():
    g = torch.Generator().manual_seed(6)
    P = 20
    honest = torch.randn(6, 1, P, generator=g)
    bad = torch.randn(4, 1, P, generator=g) + 1e6
    up = torch.cat([bad[:2], honest[:3], bad[2:], honest[3:]])
    theta = torch.zeros(1, P)
    ref.geomed_aggregate_slots_(theta, up, torch.ones(10, 1))
    h = honest[:, 0].double()
    diam = torch.cdist(h, h).max()
    assert torch.linalg.norm(theta[0].double() - h.mean(0)) <= diam
    mean = torch.zeros(1, P)
    ref.cluster_aggregate_(mean, up, torch.ones(10, 1))
    assert torch.linalg.norm(mean[0].double() - h.mean(0)) > 1e5


def test_edge_cases():
    g = torch.Generator().manual_seed(8)
    up = torch.randn(5, 1, 7, generator=g)
    one = torch.zeros(1, 7)
    ref.geomed_aggregate_slots_(one, up[1:2], torch.ones(1, 1))
    assert torch.equal(one[0], up[1, 0])                       # n = 1: exact copy
    two, med = torch.zeros(1, 7), torch.zeros(1, 7)
    ref.geomed_aggregate_slots_(two, up[:2], torch.ones(2, 1))
    ref.robust_aggregate_slots_(med, up[:2], torch.ones(2, 1), "median")
    assert _same(two, med)                                      # n = 2: exactly the K19 median
    inf = up.clone()
    inf[2, 0, 3] = float("inf")                                 # d = +inf: weight 0, left out of the sum
    got = torch.zeros(1, 7)
    ref.geomed_aggregate_slots_(got, inf, torch.ones(5, 1))
    assert torch.isfinite(got).all() and _close(got, weiszfeld(torch.zeros(1, 7), inf, torch.ones(5, 1)))
    nan = up.clone()
    nan[4, 0, 0] = float("nan")                                 # a NaN distance: the whole slot is NaN
    got = torch.zeros(1, 7)
    ref.geomed_aggregate_slots_(got, nan, torch.ones(5, 1))
    assert (got.view(torch.int32) == 0x7FC00000).all()
    w0 = torch.randn(3, 1, 3, generator=g)
    for i in range(3):                                          # every row has an infinite distance: W = 0 keeps v⁰
        w0[i, 0, i] = float("inf")
    got, med = torch.zeros(1, 3), torch.zeros(1, 3)
    ref.geomed_aggregate_slots_(got, w0, torch.ones(3, 1))
    ref.robust_aggregate_slots_(med, w0, torch.ones(3, 1), "median")
    assert _same(got, med) and torch.isfinite(got).all()


def test_geomed_params():
    assert ref.geomed_params(4, 1e-6) == (4, 1e-6)
    assert ref.geomed_params(np.int64(100), 1) == (100, 1.0)
    for it, nu in [(0, 1e-6), (101, 1e-6), (True, 1e-6), (4.0, 1e-6), (4, 0.0), (4, -1.0), (4, float("nan")),
                   (4, float("inf")), (4, True), (4, "x")]:
        with pytest.raises(ValueError):
            ref.geomed_params(it, nu)
    assert "geometric_median" in ref.AGGREGATION_RULES
    assert ref.aggregation_params("geometric_median", 0.1) == ("geometric_median", 0.1)


def test_ops_dispatch_and_server_optimizer_on_cpu():
    from feddrift_b200.ops.server_opt import SlotServerOpt
    bank, up, n = _arena(7, M=3, P=11, seed=2)
    n[:, 2] = 0
    rule = ("geometric_median", 0.1, 3, 1e-6)
    plain = bank.clone()
    assert torch.equal(ops.cluster_aggregate_(plain, up, n, None, rule), (n > 0).sum(0).float())
    want = bank.clone()
    ref.geomed_aggregate_slots_(want, up, n, 3, 1e-6)
    assert _same(plain, want)
    so = SlotServerOpt("adam", 3, 11, "cpu", lr=0.1)
    th = bank.clone()
    ops.cluster_aggregate_(th, up, n, so, rule)
    want = bank.clone()
    s0, s1, st = torch.zeros(3, 11), torch.zeros(3, 11), torch.zeros(3, dtype=torch.int32)
    ref.server_opt_slots_(want, plain, torch.tensor([True, True, False]), "adam", s0, s1, st, 0.1)
    assert torch.equal(th, want) and torch.equal(so.s0, s0) and so.step.tolist() == [1, 1, 0]


def test_oracle_round_applies_the_rule_after_compression_and_defense():
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    n = _weights(st)
    kw = dict(compression="qsgd", quantize_level=4, quantize_bucket=8, defense="weak_dp", norm_bound=0.05, stddev=0.01)
    r = dict(copy.deepcopy(st), aggregation_rule="geometric_median", geomed_iters=3, geomed_nu=1e-5, **kw)
    r["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(r, 1)
    up = r["client_out"].clone()
    ref.robust_clip_slots_(up, theta0, n, 0.05, None, 0.01, ref.defense_seed(st["seed"], 0))
    want = theta0.clone()
    ref.geomed_aggregate_slots_(want, up, n, 3, 1e-5)
    assert _same(r["theta"], want)


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


def test_drift_sim_fused_and_generic_routes_agree():
    args = _sea(aggregation_rule="geometric_median", geomed_iters=5, geomed_nu=1e-5)
    fused, _ = _run(args, end=2)
    generic, _ = _run(copy.deepcopy(args), end=2, generic=True)
    assert fused.agg_rule == ("geometric_median", 0.1, 5, 1e-5)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    med, _ = _run(_sea(aggregation_rule="median"), end=2)
    assert med.agg_rule == ("median", 0.1)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, med.bank.theta)


def test_generic_route_passes_the_trainable_mask(monkeypatch):
    calls = []
    real = ops.cluster_aggregate_

    def wrapped(theta, cp, n, server_opt=None, rule=None, mask=None):
        calls.append((theta.clone(), cp.clone(), n.clone(), rule, mask))
        return real(theta, cp, n, server_opt, rule, mask)
    monkeypatch.setattr(ops, "cluster_aggregate_", wrapped)
    sim = DriftSim(make_args(model="cnn", dataset="MNIST", client_num_in_total=5, concept_num=2, concept_drift_algo="win-1",
                             concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=1,
                             total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05,
                             aggregation_rule="geometric_median", geomed_iters=2),
                   device="cpu", sink=MetricsSink())
    sim.begin_time_step(0)
    sim.run_rounds(1)
    theta0, cp, n, rule, mask = calls[0]
    assert rule == ("geometric_median", 0.1, 2, 1e-6)
    assert (mask is None and sim.defense_mask is None) or torch.equal(mask, sim.defense_mask)
    want = theta0.clone()
    ref.geomed_aggregate_slots_(want, cp, n, 2, 1e-6, mask)
    assert _same(sim.bank.theta, want)


def test_checkpoint_resume_with_geomed(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, aggregation_rule="geometric_median", geomed_iters=3)
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
                          _sea(aggregation_rule="geometric_median", geomed_iters=6, client_num_in_total=W))
    assert agg.agg_rule == ("geometric_median", 0.1, 6, 1e-6)
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
    want = theta0.clone()
    ref.geomed_aggregate_slots_(want, raw, agg.upload_n.clone(), 6, 1e-6)
    assert _same(agg.bank.theta, want)


def test_facade_inproc_matches_the_engine():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args, run_device, run_facade
    from feddrift_b200.utils.metrics import set_sink
    base = ["--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60", "--aggregation_rule", "geometric_median"]
    p = add_args(argparse.ArgumentParser())
    sf, se, sm = MetricsSink(), MetricsSink(), MetricsSink()
    f = run_facade(p.parse_args(["--engine", "facade"] + base), set_sink(sf))
    run_device(p.parse_args(["--engine", "device"] + base), set_sink(se))
    run_facade(p.parse_args(["--engine", "facade", "--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60"]),
               set_sink(sm))
    assert len(f["history"]) == 2
    assert np.allclose(sf.series("Test/Acc"), se.series("Test/Acc"), atol=0.02)
    assert sf.series("Train/Loss") != sm.series("Train/Loss")


@pytest.mark.parametrize("kw", [dict(aggregation_rule="krum"), dict(aggregation_rule="geometric_median", geomed_iters=0),
                                dict(aggregation_rule="geometric_median", geomed_iters=101),
                                dict(aggregation_rule="mean", geomed_iters=True),
                                dict(aggregation_rule="geometric_median", geomed_nu=float("nan")),
                                dict(aggregation_rule="median", geomed_nu=0.0),
                                dict(aggregation_rule="geometric_median", geomed_nu=-1e-6)])
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
    sim = DriftSim(_sea(aggregation_rule="geometric_median"), device="cpu", sink=MetricsSink())
    from feddrift_b200.parallel.symm import attach_multi_gpu
    with pytest.raises(ValueError, match="aggregation_rule"):
        attach_multi_gpu(sim, 2, 0)
    sim.shard_clients = True
    with pytest.raises(ValueError, match="aggregation_rule"):
        sim.run_time_step(0)
    sim2 = DriftSim(_sea(aggregation_rule="geometric_median"), device="cpu", sink=MetricsSink())
    sim2.multi = {"world": 2}
    with pytest.raises(ValueError, match="aggregation_rule"):
        sim2.run_time_step(0)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.geomed_iters, a.geomed_nu) == (4, 1e-6)
    assert (make_args().geomed_iters, make_args().geomed_nu) == (4, 1e-6)
    a = p.parse_args(["--aggregation_rule", "geometric_median", "--geomed_iters", "10", "--geomed_nu", "1e-4"])
    assert (a.aggregation_rule, a.geomed_iters, a.geomed_nu) == ("geometric_median", 10, 1e-4)
    with pytest.raises(SystemExit):
        p.parse_args(["--aggregation_rule", "krum"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2g_sea_fnn_100clients_geomed_feddrift"]
    assert cfg["aggregation_rule"] == "geometric_median" and cfg["client_num_in_total"] == 100


# thresholds fixed from the CPU run of test_robust_agg's Byzantine scenario (honest clients' mean Test/Acc after the last
# round: geometric median ≈ 0.69, mean 0.60)
GEOMED_MIN = 0.67


def test_byzantine_clients_geometric_median_holds():
    gm, sim = honest_test_acc("geometric_median")
    mean, _ = honest_test_acc("mean")
    assert sim.agg_rule[0] == "geometric_median" and BYZ == 3
    assert gm >= GEOMED_MIN, (gm, mean)
    assert mean <= MEAN_MAX, (gm, mean)
