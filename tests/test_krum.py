"""Multi-Krum cluster aggregation (``--aggregation_rule multi_krum``) of the continual engines on the CPU: the oracle against
an independent brute force, a hand-computed example, non-finite rows, the distance mask, client permutations, the
parameters, the server optimizer, the oracle round's order of operations, the device engine's two routes, checkpoint
resume, the façade, the rejected configurations, the CLI and the Byzantine scenario."""
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
from test_robust_agg import BYZ, BYZ_KW, MEAN_MAX, _same, byzantine_data
from test_robust_defense import _weights


def brute_krum(theta, uploads, n, f=1, m=1, mask=None):
    """Independent definition with python loops: float64 numpy distances of the fp32 differences, sorted lists for the
    scores and the selection, fp32 numpy sums in client order and one fp32 division."""
    out = theta.clone()
    X = uploads.numpy()
    C, M, P = X.shape
    keep = np.ones(P) if mask is None else mask.numpy().astype(np.float64)
    for s in range(M):
        rows = [c for c in range(C) if float(n[c, s]) > 0]
        k = len(rows)
        if k == 0:
            continue
        sel = [0]
        if k > 1:
            D = [[0.0] * k for _ in range(k)]
            for i in range(k):
                for j in range(k):
                    if i != j:
                        diff = (X[rows[i], s] - X[rows[j], s]).astype(np.float64)
                        with np.errstate(invalid="ignore", over="ignore"):
                            d = float(np.sum(np.where(keep > 0, diff * diff, 0.0)))
                        D[i][j] = np.inf if np.isnan(d) else d
            nb = min(max(k - f - 2, 1), k - 1)
            scores = []
            for i in range(k):
                near = sorted((D[i][j], j) for j in range(k) if j != i)
                scores.append(sum(d for d, _ in near[:nb]))
            ranked = sorted(range(k), key=lambda i: (scores[i], i))
            sel = sorted(ranked[:min(m, k)])
        with np.errstate(invalid="ignore", over="ignore"):
            v = X[rows[sel[0]], s].copy()
            for i in sel[1:]:
                v = (v + X[rows[i], s]).astype(np.float32)
            if len(sel) > 1:
                v = (v / np.float32(len(sel))).astype(np.float32)
        out[s, :P] = torch.from_numpy(v)
    return out


def _arena(C, M=3, P=13, pad=0, seed=0):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, P + pad, generator=g)
    up = torch.randn(C, M, P, generator=g) * (1.0 + torch.arange(C, dtype=torch.float32)[:, None, None] / 3)
    n = (torch.rand(C, M, generator=g) * 5).floor() + (torch.arange(C) % 2)[:, None]
    return bank, up, n


@pytest.mark.parametrize("C", [1, 2, 3, 7, 10])
@pytest.mark.parametrize("f", [0, 1, 3, 1000])
@pytest.mark.parametrize("m", ["1", "2", "n-f", "over"])
def test_oracle_matches_brute_force(C, f, m):
    bank, up, n = _arena(C, pad=3, seed=C + 10 * f)
    n[:, 1] = 0                                          # a slot without participants keeps its model
    k = int((n[:, 0] > 0).sum())
    mm = {"1": 1, "2": 2, "n-f": max(1, k - f), "over": C + 5}[m]
    want = brute_krum(bank, up, n, f, mm)
    got = bank.clone()
    counts = ref.krum_aggregate_slots_(got[:, :13], up, n, f, mm)
    assert _same(got, want), (got - want).abs().max()
    assert torch.equal(got[1], bank[1]) and torch.equal(got[:, 13:], bank[:, 13:])
    assert torch.equal(counts, (n > 0).sum(0).float())


def test_m1_is_one_upload_bit_for_bit():
    bank, up, n = _arena(9, M=2, P=31, seed=4)
    n[:] = 1
    got = bank.clone()
    ref.krum_aggregate_slots_(got, up, n, 2, 1)
    for s in range(2):
        assert any(torch.equal(got[s].view(torch.int32), up[c, s].view(torch.int32)) for c in range(9))


def test_hand_computed_five_points():
    pts = torch.tensor([[0.0, 0.0], [1.0, 0.0], [0.0, 1.0], [1.0, 1.0], [10.0, 10.0]])
    D = [[float(((pts[i] - pts[j]) ** 2).sum()) for j in range(5)] for i in range(5)]
    # n = 5, f = 1: k = 2 neighbours; each corner of the unit square has two at distance² 1, the far point 162 and 181
    scores, sel = ref.krum_select(D, 1, 1)
    assert scores == [2.0, 2.0, 2.0, 2.0, 343.0] and sel == [0]   # a four-way tie goes to the lowest client
    assert ref.krum_select(D, 1, 4)[1] == [0, 1, 2, 3]
    assert ref.krum_select(D, 1, 5)[1] == [0, 1, 2, 3, 4]
    up = pts[:, None, :]
    theta = torch.zeros(1, 2)
    ref.krum_aggregate_slots_(theta, up, torch.ones(5, 1), 1, 4)
    assert theta.tolist() == [[0.5, 0.5]]                         # the far upload stays out of the average
    perm = up[[4, 3, 2, 1, 0]]
    ref.krum_aggregate_slots_(theta, perm, torch.ones(5, 1), 1, 1)
    assert theta.tolist() == [[1.0, 1.0]]                         # the tie now goes to (1, 1), client 1
    assert ref.krum_neighbours(5, 1) == 2 and ref.krum_neighbours(5, 0) == 3 and ref.krum_neighbours(5, 9) == 1
    assert ref.krum_neighbours(2, 0) == 1


def test_non_finite_rows_and_the_mask():
    g = torch.Generator().manual_seed(8)
    up = torch.randn(6, 1, 9, generator=g)
    bad = up.clone()
    bad[1, 0, 3] = float("nan")
    bad[4, 0, 0] = float("inf")
    for m in (1, 2, 4):
        got = torch.zeros(1, 9)
        ref.krum_aggregate_slots_(got, bad, torch.ones(6, 1), 1, m)
        assert torch.isfinite(got).all()
        assert _same(got, brute_krum(torch.zeros(1, 9), bad, torch.ones(6, 1), 1, m))
    got = torch.zeros(1, 9)                                       # m_eff = n: the non-finite rows are selected too
    ref.krum_aggregate_slots_(got, bad, torch.ones(6, 1), 1, 6)
    assert torch.isnan(got[0, 3]) and not torch.isfinite(got[0, 0])
    # the mask keeps the masked entries out of the distances but in the average
    mask = torch.arange(9) % 4 != 1
    big = up.clone()
    big[0, 0, ~mask] += 1e6                                       # far only in masked entries: still selectable
    got = torch.zeros(1, 9)
    ref.krum_aggregate_slots_(got, big, torch.ones(6, 1), 1, 6, mask)
    assert _same(got, brute_krum(torch.zeros(1, 9), big, torch.ones(6, 1), 1, 6, mask))
    assert (got[0, ~mask] > 1e5).all()                            # the masked entries are averaged
    for m in (1, 2, 3):
        a, b = torch.zeros(1, 9), torch.zeros(1, 9)
        ref.krum_aggregate_slots_(a, big, torch.ones(6, 1), 1, m, mask)
        ref.krum_aggregate_slots_(b, up, torch.ones(6, 1), 1, m, mask)
        assert _same(a, brute_krum(torch.zeros(1, 9), big, torch.ones(6, 1), 1, m, mask))
        assert _same(a[0, mask], b[0, mask])                       # same distances, so the same selection
    unmasked = torch.zeros(1, 9)
    ref.krum_aggregate_slots_(unmasked, big, torch.ones(6, 1), 1, 5)
    assert (unmasked.abs() < 1e3).all()                            # without the mask row 0 is far and left out
    nanmask = up.clone()
    nanmask[2, 0, 1] = float("nan")                               # a NaN in a masked-out entry: row 2 may be selected
    got = torch.zeros(1, 9)
    ref.krum_aggregate_slots_(got, nanmask, torch.ones(6, 1), 1, 6, mask)
    assert torch.isnan(got[0, 1]) and torch.isfinite(got[0, mask]).all()


def test_client_permutation():
    bank, up, n = _arena(10, M=2, P=21, seed=6)
    n[:] = 1
    perm = torch.randperm(10, generator=torch.Generator().manual_seed(1))
    for m in (1, 3):
        a, b = bank.clone(), bank.clone()
        ref.krum_aggregate_slots_(a, up, n, 2, m)
        ref.krum_aggregate_slots_(b, up[perm], n, 2, m)
        if m == 1:
            assert _same(a, b)
        else:
            assert torch.allclose(a, b, rtol=1e-6, atol=1e-6)


def test_krum_params():
    assert ref.krum_params(1, 1) == (1, 1)
    assert ref.krum_params(np.int64(0), 65535) == (0, 65535)
    for f, m in [(-1, 1), (65536, 1), (True, 1), (1.0, 1), ("1", 1), (1, 0), (1, 65536), (1, False), (1, 2.0), (None, 1)]:
        with pytest.raises(ValueError):
            ref.krum_params(f, m)
    assert "multi_krum" in ref.AGGREGATION_RULES and "krum" not in ref.AGGREGATION_RULES
    assert ref.aggregation_params("multi_krum", 0.1) == ("multi_krum", 0.1)
    with pytest.raises(ValueError):
        ref.aggregation_params("krum", 0.1)


def test_ops_dispatch_and_server_optimizer_on_cpu():
    from feddrift_b200.ops.server_opt import SlotServerOpt
    bank, up, n = _arena(7, M=3, P=11, seed=2)
    n[:, 2] = 0
    rule = ("multi_krum", 0.1, 1, 2)
    plain = bank.clone()
    assert torch.equal(ops.cluster_aggregate_(plain, up, n, None, rule), (n > 0).sum(0).float())
    want = bank.clone()
    ref.krum_aggregate_slots_(want, up, n, 1, 2)
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
    r = dict(copy.deepcopy(st), aggregation_rule="multi_krum", krum_f=1, krum_m=2, **kw)
    r["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(r, 1)
    up = r["client_out"].clone()
    ref.robust_clip_slots_(up, theta0, n, 0.05, None, 0.01, ref.defense_seed(st["seed"], 0))
    want = theta0.clone()
    ref.krum_aggregate_slots_(want, up, n, 1, 2)
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
    args = _sea(aggregation_rule="multi_krum", krum_f=1, krum_m=2)
    fused, _ = _run(args, end=2)
    generic, _ = _run(copy.deepcopy(args), end=2, generic=True)
    assert fused.agg_rule == ("multi_krum", 0.1, 1, 2)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    mean, _ = _run(_sea(), end=2)
    assert mean.agg_rule is None
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, mean.bank.theta)


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
                             aggregation_rule="multi_krum", krum_f=0, krum_m=2),
                   device="cpu", sink=MetricsSink())
    sim.begin_time_step(0)
    sim.run_rounds(1)
    theta0, cp, n, rule, mask = calls[0]
    assert rule == ("multi_krum", 0.1, 0, 2)
    assert (mask is None and sim.defense_mask is None) or torch.equal(mask, sim.defense_mask)
    want = theta0.clone()
    ref.krum_aggregate_slots_(want, cp, n, 0, 2, mask)
    assert _same(sim.bank.theta, want)


def test_checkpoint_resume_with_multi_krum(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, aggregation_rule="multi_krum", krum_f=1, krum_m=3)
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
                          _sea(aggregation_rule="multi_krum", krum_f=1, krum_m=2, client_num_in_total=W))
    assert agg.agg_rule == ("multi_krum", 0.1, 1, 2)
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
    ref.krum_aggregate_slots_(want, raw, agg.upload_n.clone(), 1, 2)
    assert _same(agg.bank.theta, want)


def test_facade_inproc_matches_the_engine():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args, run_device, run_facade
    from feddrift_b200.utils.metrics import set_sink
    base = ["--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60", "--aggregation_rule", "multi_krum",
            "--krum_m", "2"]
    p = add_args(argparse.ArgumentParser())
    sf, se, sm = MetricsSink(), MetricsSink(), MetricsSink()
    f = run_facade(p.parse_args(["--engine", "facade"] + base), set_sink(sf))
    run_device(p.parse_args(["--engine", "device"] + base), set_sink(se))
    run_facade(p.parse_args(["--engine", "facade", "--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60"]),
               set_sink(sm))
    assert len(f["history"]) == 2
    assert np.allclose(sf.series("Test/Acc"), se.series("Test/Acc"), atol=0.02)
    assert sf.series("Train/Loss") != sm.series("Train/Loss")


@pytest.mark.parametrize("kw", [dict(aggregation_rule="krum"), dict(aggregation_rule="multi_krum", krum_f=-1),
                                dict(aggregation_rule="multi_krum", krum_m=0),
                                dict(aggregation_rule="mean", krum_f=True),
                                dict(aggregation_rule="median", krum_m=1.5),
                                dict(aggregation_rule="multi_krum", krum_m=65536)])
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
    sim = DriftSim(_sea(aggregation_rule="multi_krum"), device="cpu", sink=MetricsSink())
    from feddrift_b200.parallel.symm import attach_multi_gpu
    with pytest.raises(ValueError, match="aggregation_rule"):
        attach_multi_gpu(sim, 2, 0)
    sim.shard_clients = True
    with pytest.raises(ValueError, match="aggregation_rule"):
        sim.run_time_step(0)
    sim2 = DriftSim(_sea(aggregation_rule="multi_krum"), device="cpu", sink=MetricsSink())
    sim2.multi = {"world": 2}
    with pytest.raises(ValueError, match="aggregation_rule"):
        sim2.run_time_step(0)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.krum_f, a.krum_m) == (1, 1)
    assert (make_args().krum_f, make_args().krum_m) == (1, 1)
    a = p.parse_args(["--aggregation_rule", "multi_krum", "--krum_f", "3", "--krum_m", "4"])
    assert (a.aggregation_rule, a.krum_f, a.krum_m) == ("multi_krum", 3, 4)
    with pytest.raises(SystemExit):
        p.parse_args(["--aggregation_rule", "krum"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2k_sea_fnn_100clients_multikrum_feddrift"]
    assert cfg["aggregation_rule"] == "multi_krum" and cfg["client_num_in_total"] == 100
    sim = DriftSim(make_args(**dict(cfg, comm_round=1, total_train_iteration=1)), device="cpu", sink=MetricsSink())
    assert sim.agg_rule == ("multi_krum", 0.1, 1, 1)


# ----------------------------------------------------------------------------- Byzantine scenario
# test_robust_agg's scenario (clients 0..2 of 10 flip their labels and scale their features by 100) with f = BYZ.
# Threshold fixed from the CPU run (honest clients' mean Test/Acc after the last round: multi_krum f = 3 ≈ 0.68 with m = 1
# and 0.69 with m = 3, mean 0.60, the majority class), with a little room for the fused kernel's last-bit differences
KRUM_MIN = 0.66


def krum_honest_test_acc(device="cpu", f=BYZ, m=1):
    sim = DriftSim(make_args(aggregation_rule="multi_krum", krum_f=f, krum_m=m, **BYZ_KW), data=byzantine_data(), device=device,
                   sink=MetricsSink())
    sim.run()
    accs = [sim.sink.series(f"Test/Acc-CL-{c}")[-1] for c in range(BYZ, 10)]
    return float(np.mean(accs)), sim


def test_byzantine_clients_multi_krum_holds():
    from test_robust_agg import honest_test_acc
    kr, sim = krum_honest_test_acc()
    kr3, _ = krum_honest_test_acc(m=3)
    mean, _ = honest_test_acc("mean")
    assert sim.agg_rule == ("multi_krum", 0.1, BYZ, 1)
    assert kr >= KRUM_MIN and kr3 >= KRUM_MIN, (kr, kr3, mean)
    assert mean <= MEAN_MAX, (kr, kr3, mean)
