"""Simulated Byzantine clients (``--attack_type`` sign_flip / gaussian / alie / ipm) of the continual engines on the CPU: the
oracle against an independent numpy-loop definition, the attacker set, a = 0 against no attack, the oracle round's order of
operations, the device engine's two routes, honest-only metrics, checkpoint resume, the façade, the rejected
configurations, the CLI and a Byzantine scenario on clean data."""
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
from test_robust_agg import BYZ, BYZ_KW, _same
from test_robust_defense import _weights

KINDS = ["sign_flip", "gaussian", "alie", "ipm"]


def np_attack(rows, theta, n, att, kind, s, mask=None, seed=0):
    """Independent definition with python loops over numpy float32 scalars (each operation rounded on its own)."""
    X = rows.numpy().copy()
    C, M, P = X.shape
    th = theta.numpy()[:, :P]
    s = np.float32(s)
    keep = np.ones(P, dtype=bool) if mask is None else mask.numpy().astype(bool)
    for m in range(M):
        bad = [c for c in range(C) if att[c] and float(n[c, m]) > 0]
        good = [c for c in range(C) if not att[c] and float(n[c, m]) > 0]
        if not bad or (kind in ("alie", "ipm") and not good):
            continue
        h = np.float32(len(good))
        for e in range(P):
            if not keep[e]:
                continue
            t = np.float32(th[m, e])
            if kind in ("alie", "ipm"):
                acc = np.float32(0.0)
                for c in good:
                    acc = np.float32(acc + X[c, m, e])
                mu = np.float32(acc / h)
                if kind == "alie":
                    ss = np.float32(0.0)
                    for c in good:
                        d = np.float32(rows[c, m, e].item() - mu)
                        ss = np.float32(ss + np.float32(d * d))
                    v = np.float32(mu - np.float32(s * np.float32(np.sqrt(np.float32(ss / h)))))
                else:
                    v = np.float32(t - np.float32(s * np.float32(mu - t)))
            for c in bad:
                x = np.float32(X[c, m, e])
                if kind == "sign_flip":
                    X[c, m, e] = np.float32(t - np.float32(s * np.float32(x - t)))
                elif kind == "gaussian":
                    xi = np.float32(ref.gauss_hash_rows(seed, [c * M + m], P)[0, e].item())
                    X[c, m, e] = np.float32(t + np.float32(s * xi))
                else:
                    X[c, m, e] = v
    return torch.from_numpy(X)


def _arena(C=9, M=4, P=13, pad=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(M, P + pad, generator=g)
    rows = theta[None, :, :P] + torch.randn(C, M, P, generator=g) * (1.0 + torch.arange(C, dtype=torch.float32)[:, None, None])
    n = (torch.rand(C, M, generator=g) * 4).floor() + 1
    return theta, rows, n


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("masked", [False, True])
def test_oracle_matches_the_numpy_definition(kind, masked):
    theta, rows, n = _arena(seed=3)
    C, M, P = rows.shape
    att = torch.zeros(C, dtype=torch.bool)
    att[[1, 4, 6]] = True
    n[:, 0] = 0
    n[1, 0] = 2                        # slot 0: one attacker, no honest participant (h = 0)
    n[:, 1] = 0
    n[[1, 2], 1] = 3                   # slot 1: h = 1
    n[4, 2] = 0                        # slot 2: an attacker that did not train stays as it is
    mask = (torch.arange(P) % 5 != 2) if masked else None
    seed = ref.attack_seed(7, 2)
    want = np_attack(rows, theta, n, att.tolist(), kind, 2.5, mask, seed)
    got = rows.clone()
    ref.attack_slots_(got, theta, n, att, kind, 2.5, mask, seed)
    assert _same(got, want), (got - want).abs().max()
    assert torch.equal(got[~att], rows[~att])                    # honest rows are untouched
    assert torch.equal(got[4, 2], rows[4, 2])                    # n = 0
    if masked:
        assert torch.equal(got[:, :, ~mask], rows[:, :, ~mask])  # BatchNorm-like entries keep the attacker's values
    if kind in ("alie", "ipm"):
        assert torch.equal(got[1, 0], rows[1, 0])                # h = 0: left as trained
        on = torch.ones(P, dtype=torch.bool) if mask is None else mask
        assert torch.equal(got[1, 3, on], got[6, 3, on]) and torch.equal(got[4, 3, on], got[6, 3, on])   # colluders agree
    else:
        assert not torch.equal(got[1, 0], rows[1, 0])


def test_alie_deviation_is_correctly_rounded():
    """σ = sqrt_rn(...): checked over many entries against numpy's float32 arrays (IEEE sqrt)."""
    theta, rows, n = _arena(C=6, M=1, P=1 << 16, pad=0, seed=12)
    n[:] = 1
    att = torch.tensor([False, True, False, False, True, False])
    got = rows.clone()
    ref.attack_slots_(got, theta, n, att, "alie", 0.75)
    X = rows.numpy()[:, 0]
    good = [0, 2, 3, 5]
    h = np.float32(len(good))
    acc = np.zeros(X.shape[1], np.float32)
    for c in good:
        acc = (acc + X[c]).astype(np.float32)
    mu = (acc / h).astype(np.float32)
    ss = np.zeros_like(mu)
    for c in good:
        d = (X[c] - mu).astype(np.float32)
        ss = (ss + (d * d).astype(np.float32)).astype(np.float32)
    v = (mu - (np.float32(0.75) * np.sqrt((ss / h).astype(np.float32))).astype(np.float32)).astype(np.float32)
    assert _same(got[1, 0], torch.from_numpy(v)) and _same(got[4, 0], torch.from_numpy(v))


@pytest.mark.parametrize("kind", KINDS)
def test_all_clients_attacking(kind):
    theta, rows, n = _arena(C=5, M=2, P=7, seed=5)
    att = torch.ones(5, dtype=torch.bool)
    got = rows.clone()
    ref.attack_slots_(got, theta, n, att, kind, 0.5, None, 11)
    assert _same(got, np_attack(rows, theta, n, [True] * 5, kind, 0.5, None, 11))
    if kind in ("alie", "ipm"):
        assert torch.equal(got, rows)                            # no honest upload to craft from


def test_hand_computed_values():
    theta = torch.zeros(1, 1)
    rows = torch.tensor([[[1.0]], [[3.0]], [[5.0]]])
    n = torch.ones(3, 1)
    att = torch.tensor([False, False, True])
    for kind, s, want in [("sign_flip", 2.0, -10.0), ("alie", 1.0, 1.0), ("ipm", 0.5, -1.0)]:
        got = rows.clone()
        ref.attack_slots_(got, theta, n, att, kind, s)
        assert got[2, 0, 0].item() == want and got[:2].tolist() == rows[:2].tolist()


def test_attacker_clients():
    a5 = ref.attacker_clients(40, 5, 3)
    assert a5.dtype == torch.bool and int(a5.sum()) == 5
    assert torch.equal(a5, ref.attacker_clients(40, 5, 3))
    prev = torch.zeros(40, dtype=torch.bool)
    for a in range(41):
        cur = ref.attacker_clients(40, a, 3)
        assert int(cur.sum()) == a and bool((cur | ~prev).all())  # nested: the set for a contains the one for a − 1
        prev = cur
    assert not torch.equal(a5, ref.attacker_clients(40, 5, 4))
    kw = dict(client_num_in_total=10, comm_round=3, total_train_iteration=2, sample_num=40, epochs=2, attack_type="sign_flip",
              attack_clients=3, dummy_arg=2)
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    sampled = DriftSim(make_args(client_num_per_round=4, **kw), device="cpu", sink=MetricsSink())
    assert torch.equal(full.attackers, ref.attacker_clients(10, 3, 2)) and torch.equal(sampled.attackers, full.attackers)
    full.run()
    assert torch.equal(full.attackers, ref.attacker_clients(10, 3, 2))


def test_attack_params():
    assert ref.attack_params("alie", 3, 1.5, 10) == ("alie", 3, 1.5)
    assert ref.attack_params(None, np.int64(0), 1, 4) == ("none", 0, 1.0)
    for t, a, s in [("krum", 1, 1.0), ("alie", -1, 1.0), ("alie", 11, 1.0), ("alie", True, 1.0), ("alie", 1.0, 1.0),
                    ("alie", 1, 0.0), ("alie", 1, -1.0), ("alie", 1, float("inf")), ("alie", 1, float("nan")), ("alie", 1, 1e39),
                    ("alie", 1, 1e-50), ("alie", 1, "x"), ("alie", 1, True)]:
        with pytest.raises(ValueError):
            ref.attack_params(t, a, s, 10)
    assert ref.attack_seed(5, 1) not in (ref.defense_seed(5, 1), ref.compress_seed(5, 1))


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


@pytest.mark.parametrize("kind", KINDS)
def test_zero_attackers_is_no_attack(kind):
    plain, po = _run(_sea(), end=2)
    zero, zo = _run(_sea(attack_type=kind, attack_clients=0, attack_scale=3.0), end=2)
    assert zero.attack is None and not bool(zero.attackers.any())
    assert _same(zero.bank.theta, plain.bank.theta) and zo["history"] == po["history"]
    assert zero.sink.series("Test/Acc") == plain.sink.series("Test/Acc")


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_round_applies_the_attack_after_compression_and_before_defense_and_rule(kind):
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    n = _weights(st)
    att = torch.zeros(C, dtype=torch.bool)
    att[[2, 5]] = True
    kw = dict(compression="qsgd", quantize_level=4, quantize_bucket=8, defense="norm_diff_clipping", norm_bound=0.5)
    plain = dict(copy.deepcopy(st), **kw)
    plain["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(plain, 1)
    r = dict(copy.deepcopy(st), aggregation_rule="median", attack_type=kind, attack_clients=2, attack_scale=3.0, attackers=att, **kw)
    r["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(r, 1)
    up = plain["client_out"].clone()                               # the compressed uploads
    ref.attack_slots_(up, theta0, n, att, kind, 3.0, None, ref.attack_seed(st["seed"], 0))
    assert _same(r["client_out"], up)                             # client_out sees the attacked uploads
    ref.robust_clip_slots_(up, theta0, n, 0.5, None, 0.0, 0)
    want = theta0.clone()
    ref.robust_aggregate_slots_(want, up, n, "median")
    assert _same(r["theta"], want)


@pytest.mark.parametrize("kind", KINDS)
def test_drift_sim_fused_and_generic_routes_agree(kind):
    args = _sea(attack_type=kind, attack_clients=3, attack_scale=2.0)
    fused, _ = _run(args, end=2)
    generic, _ = _run(copy.deepcopy(args), end=2, generic=True)
    assert fused.attack == (kind, 2.0)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    clean, _ = _run(_sea(), end=2)
    assert not torch.allclose(fused.bank.theta, clean.bank.theta)


def test_honest_accuracy_metrics():
    sim, out = _run(_sea(attack_type="sign_flip", attack_clients=3, attack_scale=4.0))
    att = sim.attackers.numpy()
    t = sim.t
    n_test = sim.data_host.nsamp[t + 1].numpy().astype(np.float64)
    accs = np.array([sim.sink.series(f"Test/Acc-CL-{c}")[-1] for c in range(8)])
    want = float((accs[~att] * n_test[~att]).sum() / n_test[~att].sum())
    got = sim.sink.series("Test/AccHonest")[-1]
    assert abs(got - want) < 1e-9 and out["history"][-1]["test_acc_honest"] == got
    assert len(sim.sink.series("Train/AccHonest")) == len(sim.sink.series("Train/Acc"))
    res = sim.run_round()                                          # the single-round public API reports it too
    assert "test_acc_honest" in res and 0.0 <= res["test_acc_honest"] <= 1.0
    plain, pout = _run(_sea())
    assert plain.sink.series("Test/AccHonest") == [] and "test_acc_honest" not in pout["history"][-1]
    assert "test_acc_honest" not in plain.run_round()


def test_checkpoint_resume_under_an_attack(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, attack_type="gaussian", attack_clients=2, attack_scale=0.3, aggregation_rule="median")
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    full.run()
    part = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    part.run(0, 2)
    resumed = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    nxt = checkpoint.resume(resumed, checkpoint.latest(str(tmp_path)))
    assert nxt == 2
    resumed.run(nxt)
    assert _same(resumed.bank.theta, full.bank.theta)


def test_facade_aggregator_poisons_the_arena():
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    from feddrift_b200.models import utils as mutils
    M, W = 2, 6
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, W, "cpu", [model] * M, 2,
                          _sea(attack_type="alie", attack_clients=2, attack_scale=1.5, client_num_in_total=W))
    assert agg.attack == ("alie", 1.5) and int(agg.attackers.sum()) == 2
    P = agg.bank.P
    g = torch.Generator().manual_seed(3)
    agg.bank.theta.copy_(torch.randn(M, P, generator=g))
    theta0 = agg.bank.theta.clone()
    raw = theta0[None] + torch.randn(W, M, P, generator=g)
    raw[0, 1] = 0                                                    # worker 0 uploads nothing for slot 1
    order = [3, 0, 5, 1, 4, 2]                                       # worker w trains client order[w]
    agg.sample_round_clients(0, W, W)
    agg._round_clients = order
    for w in range(W):
        sds = {m: ({k: v.clone() for k, v in mutils.unflatten_to_state_dict(raw[w, m], agg.bank.spec).items()},
                   0 if (m == 1 and w == 0) else 3 + w) for m in range(M)}
        agg.add_local_trained_result(w, sds)
    assert agg.check_whether_all_receive()
    rows = torch.tensor([bool(agg.attackers[c]) for c in order])
    want = raw.clone()
    ref.attack_slots_(want, theta0, agg.upload_n, rows, "alie", 1.5)
    assert _same(agg.upload, want) and not torch.equal(agg.upload, raw)
    agg._aggregate_models()
    theta = theta0.clone()
    ref.cluster_aggregate_(theta, want, agg.upload_n.clone())
    assert torch.allclose(agg.bank.theta, theta, rtol=1e-6, atol=1e-6)


def test_facade_inproc_matches_the_engine():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args, run_device, run_facade
    from feddrift_b200.utils.metrics import set_sink
    base = ["--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60", "--attack_type", "sign_flip",
            "--attack_clients", "3", "--attack_scale", "5"]
    p = add_args(argparse.ArgumentParser())
    sf, se, sm = MetricsSink(), MetricsSink(), MetricsSink()
    f = run_facade(p.parse_args(["--engine", "facade"] + base), set_sink(sf))
    run_device(p.parse_args(["--engine", "device"] + base), set_sink(se))
    run_facade(p.parse_args(["--engine", "facade", "--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60"]),
               set_sink(sm))
    assert len(f["history"]) == 2
    assert np.allclose(sf.series("Test/Acc"), se.series("Test/Acc"), atol=0.02)
    assert sf.series("Train/Loss") != sm.series("Train/Loss")


@pytest.mark.parametrize("kw", [dict(attack_type="krum", attack_clients=1), dict(attack_type="alie", attack_clients=-1),
                                dict(attack_type="sign_flip", attack_clients=9), dict(attack_type="none", attack_clients=True),
                                dict(attack_type="ipm", attack_clients=1, attack_scale=0.0),
                                dict(attack_type="none", attack_scale=float("nan")),
                                dict(attack_type="gaussian", attack_clients=1, attack_scale=-2.0)])
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
    sim = DriftSim(_sea(attack_type="alie", attack_clients=2), device="cpu", sink=MetricsSink())
    from feddrift_b200.parallel.symm import attach_multi_gpu
    with pytest.raises(ValueError, match="attack_type"):
        attach_multi_gpu(sim, 2, 0)
    sim.shard_clients = True
    with pytest.raises(ValueError, match="attack_type"):
        sim.run_time_step(0)
    sim2 = DriftSim(_sea(attack_type="sign_flip", attack_clients=2), device="cpu", sink=MetricsSink())
    sim2.multi = {"world": 2}
    with pytest.raises(ValueError, match="attack_type"):
        sim2.run_time_step(0)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.attack_type, a.attack_clients, a.attack_scale) == ("none", 0, 1.0)
    d = make_args()
    assert (d.attack_type, d.attack_clients, d.attack_scale) == ("none", 0, 1.0)
    a = p.parse_args(["--attack_type", "ipm", "--attack_clients", "4", "--attack_scale", "0.5"])
    assert (a.attack_type, a.attack_clients, a.attack_scale) == ("ipm", 4, 0.5)
    with pytest.raises(SystemExit):
        p.parse_args(["--attack_type", "label_flip"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2a_sea_fnn_100clients_alie_median_feddrift"]
    assert (cfg["attack_type"], cfg["attack_clients"], cfg["aggregation_rule"], cfg["client_num_in_total"]) == \
        ("alie", 20, "median", 100)
    sim = DriftSim(make_args(**dict(cfg, comm_round=1, total_train_iteration=1)), device="cpu", sink=MetricsSink())
    assert sim.attack == ("alie", 1.0) and int(sim.attackers.sum()) == 20 and sim.agg_rule == ("median", 0.1)


def test_ops_dispatch_on_cpu():
    theta, rows, n = _arena(seed=9)
    att = ref.attacker_clients(rows.shape[0], 3, 1)
    for kind in KINDS:
        a, b = rows.clone(), rows.clone()
        ops.attack_slots_(a, theta, n, att, kind, 1.5, None, 4)
        ref.attack_slots_(b, theta, n, att, kind, 1.5, None, 4)
        assert _same(a, b)
    c = rows.clone()
    ops.attack_slots_(c, theta, n, att, "none", 1.5)
    assert torch.equal(c, rows)


# ----------------------------------------------------------------------------- Byzantine scenario
# test_robust_agg's federation on clean data; the BYZ clients chosen by attacker_clients upload their reversed update scaled
# by 10.  Thresholds fixed from the CPU run (honest clients' accuracy after the last round, Test/AccHonest: mean ≈ 0.42,
# median ≈ 0.69), with a margin
ATTACK_MEAN_MAX, ATTACK_MEDIAN_MIN = 0.55, 0.64


def sign_flip_honest_acc(rule, device="cpu"):
    sim = DriftSim(make_args(aggregation_rule=rule, attack_type="sign_flip", attack_clients=BYZ, attack_scale=10.0, **BYZ_KW),
                   device=device, sink=MetricsSink())
    sim.run()
    return sim.sink.series("Test/AccHonest")[-1], sim


def test_sign_flip_breaks_the_mean_and_not_the_median():
    mean, _ = sign_flip_honest_acc("mean")
    med, sim = sign_flip_honest_acc("median")
    assert int(sim.attackers.sum()) == BYZ
    assert mean <= ATTACK_MEAN_MAX, (mean, med)
    assert med >= ATTACK_MEDIAN_MIN, (mean, med)
