"""Top-k sparsification with error feedback (``--compression eftopk``) of the continual engines on the CPU: the selection
against an independent brute force, the per-entry formulas, pass-through entries and skipped rows, ρ = 1 against ``none``,
the residual's lifetime, the round oracle, the device engine's two routes, the raw-update hooks, checkpoint resume, the
façade and the rejected configurations."""
import argparse
import copy

import pytest
import torch

from feddrift_b200.models import utils as mutils
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, checkpoint, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state
from test_robust_defense import _BnNet, _weights


def _arena(C=3, M=2, P=37, pad=5, scale=0.3, seed=0, res_scale=0.05):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(M, P + pad, generator=g)   # a padded bank row
    rows = theta[None, :, :P] + scale * torch.randn(C, M, P, generator=g)
    res = res_scale * torch.randn(C, M, P, generator=g)
    return rows, theta, res


def _brute(rows, theta, res, n, k, mask=None):
    """Independent definition: python sort of (−|v| bits, index) over the trainable entries of every selected row."""
    C, M, P = rows.shape
    out_x, out_e = rows.clone(), res.clone()
    for c in range(C):
        for m in range(M):
            if n is not None and not n[c, m] > 0:
                continue
            x, th, e = rows[c, m].tolist(), theta[m, :P].tolist(), res[c, m].tolist()
            v = (rows[c, m] - theta[m, :P]) + res[c, m]
            bits = (v.view(torch.int32).to(torch.int64) & 0x7FFFFFFF).tolist()
            train = [i for i in range(P) if mask is None or bool(mask[i])]
            keep = set(sorted(train, key=lambda i: (-bits[i], i))[:k])
            for i in train:
                if i in keep:
                    out_x[c, m, i] = x[i] if e[i] == 0 else float(torch.tensor(x[i]) + torch.tensor(e[i]))
                    out_e[c, m, i] = 0.0
                else:
                    out_x[c, m, i] = th[i]
                    out_e[c, m, i] = v[i]
    return out_x, out_e


@pytest.mark.parametrize("k", [1, 5, 36, 37, 100])
@pytest.mark.parametrize("case", ["random", "ties", "zero"])
def test_oracle_matches_brute_force(k, case):
    rows, theta, res = _arena()
    if case == "ties":   # a handful of distinct magnitudes, both signs: many equal keys
        g = torch.Generator().manual_seed(4)
        mag = torch.tensor([0.0, 0.125, 0.5, 2.0])[torch.randint(0, 4, rows.shape, generator=g)]
        sgn = torch.where(torch.rand(rows.shape, generator=g) < 0.5, -1.0, 1.0)
        rows = theta[None, :, :37] + sgn * mag
        res = torch.zeros_like(rows)
    elif case == "zero":   # no update at all
        rows = theta[None, :, :37].expand(3, 2, 37).clone()
        res = torch.zeros_like(rows)
    want_x, want_e = _brute(rows, theta, res, None, min(k, 37))
    ref.eftopk_slots_(rows, theta, res, None, k)
    assert torch.equal(rows, want_x) and torch.equal(res, want_e)
    kept = (res == 0).sum(-1)
    if case == "random":
        assert bool((kept == min(k, 37)).all())


def test_entry_formulas_mask_and_skipped_rows():
    rows, theta, res = _arena(C=3, M=2, P=40)
    res[0, 0, :10] = 0.0   # kept entries with a zero residual upload x itself
    mask = torch.ones(40, dtype=torch.bool)
    mask[::3] = False
    res[..., ~mask] = 0.0
    n = torch.ones(3, 2)
    n[2, 0] = 0
    x0, e0 = rows.clone(), res.clone()
    ref.eftopk_slots_(rows, theta, res, n, 6, mask)
    want_x, want_e = _brute(x0, theta, e0, n, 6, mask)
    assert torch.equal(rows, want_x) and torch.equal(res, want_e)
    assert torch.equal(rows[..., ~mask], x0[..., ~mask]) and bool((res[..., ~mask] == 0).all())
    assert torch.equal(rows[2, 0], x0[2, 0]) and torch.equal(res[2, 0], e0[2, 0])
    th = theta[:, :40]
    for c, m in [(0, 0), (1, 1)]:
        v = (x0[c, m] - th[m]) + e0[c, m]
        kept = (res[c, m] == 0) & mask & (rows[c, m] != th[m])
        assert int(((res[c, m] == 0) & mask).sum()) >= 6
        assert torch.equal(rows[c, m][kept], torch.where(e0[c, m] == 0, x0[c, m], x0[c, m] + e0[c, m])[kept])
        dropped = mask & (res[c, m] != 0)
        assert torch.equal(rows[c, m][dropped], th[m][dropped]) and torch.equal(res[c, m][dropped], v[dropped])
        # mass is conserved: (upload − θ) + residual == v on every trainable entry, up to the rounding of x + e
        assert torch.allclose(((rows[c, m] - th[m]) + res[c, m])[mask], v[mask], rtol=0, atol=1e-6)


def test_k_rule_and_upload_bits():
    assert ref.topk_k(0.1, 30) == 3   # ⌈0.1·30⌉ is 4 in float64
    assert ref.topk_k(0.01, 37) == 1 and ref.topk_k(1.0, 37) == 37 and ref.topk_k(0.5, 5) == 3
    assert ref.topk_k(1e-9, 1000) == 1
    P = 1000
    assert ref.topk_upload_bits(P, 0, 10) == 10 * (32 + 10)
    assert ref.topk_upload_bits(1000, 24, 7) == 7 * (32 + 10) + 32 * 24
    assert ref.topk_upload_bits(1, 0, 1) == 32
    assert ref.compression_params("eftopk", 16, 512) == (0, 0)
    for bad in (0, -0.1, 1.5, float("nan"), float("inf"), "x", True):
        with pytest.raises(ValueError):
            ref.topk_ratio_param(bad)


def _with_ef(st, rho=0.3):
    return dict(st, compression="eftopk", topk_ratio=rho)


def test_oracle_round_is_the_average_of_sparsified_uploads_and_carries_the_residual():
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    plain = copy.deepcopy(st)
    plain["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(plain, 1)
    e = _with_ef(copy.deepcopy(st))
    e["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(e, 1)
    n = _weights(st)
    k = ref.topk_k(0.3, P)
    want_up, want_res = plain["client_out"].clone(), torch.zeros(C, M, P)
    ref.eftopk_slots_(want_up, theta0, want_res, n, k)
    assert torch.equal(e["client_out"], want_up) and torch.equal(e["ef_residual"], want_res)
    assert bool((want_res[n > 0] != 0).any())
    want = theta0.clone()
    ref.cluster_aggregate_(want, want_up, n)
    assert torch.allclose(e["theta"], want, rtol=0, atol=1e-6)
    for key in ("opt_m", "opt_step"):   # local training does not see the sparsification
        assert torch.equal(e[key], plain[key]), key
    # a second round starts from the residual the first one left
    e2 = copy.deepcopy(e)
    ref.fed_round_small(e2, 1)
    assert not torch.equal(e2["ef_residual"], e["ef_residual"])


def test_oracle_sparsifies_before_the_defense():
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    a = _with_ef(copy.deepcopy(st))
    a["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(a, 1)
    ad = dict(_with_ef(copy.deepcopy(st)), defense="weak_dp", norm_bound=0.1, stddev=0.01)
    ref.fed_round_small(ad, 1)
    n = _weights(st)
    up = a["client_out"].clone()
    ref.robust_clip_slots_(up, theta0, n, 0.1, None, 0.01, ref.defense_seed(st["seed"], 0))
    want = theta0.clone()
    ref.cluster_aggregate_(want, up, n)
    assert torch.allclose(ad["theta"], want, rtol=0, atol=1e-6)
    assert torch.equal(ad["ef_residual"], a["ef_residual"])


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


@pytest.mark.parametrize("generic", [False, True])
def test_ratio_one_is_bit_identical_to_none(generic):
    a, oa = _run(_sea(compression="eftopk", topk_ratio=1.0), generic=generic)
    b, ob = _run(_sea(), generic=generic)
    assert torch.equal(a.bank.theta, b.bank.theta) and oa["history"] == ob["history"]
    assert bool((a.clients.ef_res == 0).all())


def test_drift_sim_fused_and_generic_routes_agree_and_log_the_upload_size():
    args = _sea(compression="eftopk", topk_ratio=0.2)
    fused, _ = _run(args, end=2)
    generic, _ = _run(copy.deepcopy(args), end=2, generic=True)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    assert torch.allclose(generic.clients.ef_res, fused.clients.ef_res, rtol=1e-4, atol=1e-5)
    plain, _ = _run(_sea(), end=2)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, plain.bank.theta)
    P = fused.bank.P
    k = ref.topk_k(0.2, P)
    assert fused.topk_k == k
    bits = fused.sink.series("Comm/UploadBits")
    assert bits == [ref.topk_upload_bits(P, 0, k)] * 2
    assert fused.sink.series("Comm/CompressionRatio") == [32.0 * P / bits[0]] * 2
    assert fused.clients.ef_res is not None and plain.clients.ef_res is None


def test_residual_lifetime():
    sim = DriftSim(_sea(compression="eftopk", topk_ratio=0.2, concept_num=2), device="cpu", sink=MetricsSink())
    assert sim.bank.ef_res is sim.clients.ef_res
    sim.begin_time_step(0)
    sim.run_rounds(2)
    res = sim.clients.ef_res
    assert bool((res != 0).any())
    M = sim.M
    assert M >= 2
    res.fill_(0.5)
    sim.bank.copy(1, 0)   # a CFL / ClusterFL split writes a slot: its column restarts for every client
    assert bool((res[:, 1] == 0).all()) and bool((res[:, 0] == 0.5).all())
    sim.bank.copy(0, 0)
    assert bool((res[:, 0] == 0.5).all())
    sim.bank.reinit(0)
    assert bool((res[:, 0] == 0).all())
    res.fill_(0.5)
    sim.end_time_step()
    sim.begin_time_step(1)
    assert bool((sim.clients.ef_res == 0).all())


def _cnn_sim(**kw):
    d = dict(model="cnn", dataset="MNIST", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1", concept_drift_algo_arg="",
             change_points="A", sample_num=8, batch_size=8, comm_round=2, total_train_iteration=2, epochs=1, client_optimizer="sgd",
             lr=0.05)
    d.update(kw)
    sim = DriftSim(make_args(**d), device="cpu", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    return sim


def _record(monkeypatch):
    """Wrap ``ops.eftopk_slots_``: records (raw rows, residual before, n, sparsified rows) of every call."""
    from feddrift_b200 import ops
    calls = []
    real = ops.eftopk_slots_

    def wrapped(rows, theta, residual, n=None, *a, **k):
        raw, r0 = rows.clone(), residual.clone()
        out = real(rows, theta, residual, n, *a, **k)
        calls.append((raw, r0, None if n is None else n.clone(), rows.clone()))
        return out
    monkeypatch.setattr(ops, "eftopk_slots_", wrapped)
    return calls


@pytest.mark.parametrize("per_round", [4, 2])
def test_generic_cnn_round_aggregates_the_sparsified_arena(per_round, monkeypatch):
    sim = _cnn_sim(compression="eftopk", topk_ratio=0.05, client_num_per_round=per_round)
    assert sim.spec is None
    calls = _record(monkeypatch)
    theta0 = sim.bank.theta.clone()
    sim.clients.ef_res.normal_(0, 1e-3, generator=torch.Generator().manual_seed(2))
    res0 = sim.clients.ef_res.clone()
    sim.run_rounds(1)
    raw, r0, n, _ = calls[0]
    assert torch.equal(r0, res0)
    want_up, want_res = raw.clone(), res0.clone()
    ref.eftopk_slots_(want_up, theta0, want_res, n, sim.topk_k, sim.defense_mask)
    assert torch.equal(sim.clients.params, want_up) and torch.equal(sim.clients.ef_res, want_res)
    if per_round < 4:   # clients that were not sampled keep their residual
        idle = ~(n > 0).any(1)
        assert bool(idle.any())
        assert torch.equal(sim.clients.ef_res[idle], res0[idle])
    want = theta0.clone()
    ref.cluster_aggregate_(want, want_up, n)
    assert torch.allclose(sim.bank.theta, want, rtol=1e-5, atol=1e-6)


def test_batchnorm_entries_pass_through():
    from feddrift_b200.parallel.arena import ModelBank
    bank = ModelBank(_BnNet(), 2, "cpu")
    P, M, C = bank.P, 2, 3
    wmask = mutils.weight_param_mask(bank.spec)[:P].bool()
    assert not bool(wmask.all())
    g = torch.Generator().manual_seed(1)
    bank.theta.copy_(torch.randn(M, P, generator=g))
    up = bank.theta[None] + torch.randn(C, M, P, generator=g)
    res = torch.zeros(C, M, P)
    before = up.clone()
    ref.eftopk_slots_(up, bank.theta, res, torch.ones(C, M), 3, wmask)
    assert torch.equal(up[..., ~wmask], before[..., ~wmask]) and bool((res[..., ~wmask] == 0).all())
    assert int((res[..., wmask] == 0).sum()) == 3 * C * M


@pytest.mark.parametrize("algo", [("softcluster", "cfl_0.1_win-1"), ("clusterfl", "win-1")])
def test_raw_update_hooks_see_sparsified_uploads(algo, monkeypatch):
    args = _sea(concept_drift_algo=algo[0], concept_drift_algo_arg=algo[1], concept_num=2, comm_round=3,
                compression="eftopk", topk_ratio=0.1)
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    sim.begin_time_step(0)
    calls = _record(monkeypatch)
    seen = []
    if algo[0] == "clusterfl":
        sim.algo.split_round = 0
        real = sim.algo.on_client_updates
        monkeypatch.setattr(sim.algo, "on_client_updates", lambda t, p, n: (seen.append(p.clone()), real(t, p, n)))
    else:
        real = sim.algo.state.cluster_cfl
        monkeypatch.setattr(sim.algo.state, "cluster_cfl", lambda t, r, bank, p, n: (seen.append(p.clone()), real(t, r, bank, p, n))[1])
    sim.run_rounds(1)
    assert seen and calls
    raw, _, n, sparse = calls[0]
    sel = n > 0
    assert torch.equal(seen[0], sparse)
    assert not torch.equal(sparse[sel], raw[sel])


def test_checkpoint_resume_with_eftopk(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, compression="eftopk", topk_ratio=0.3)
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    full.run()
    part = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    part.run(0, 2)
    resumed = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    nxt = checkpoint.resume(resumed, checkpoint.latest(str(tmp_path)))
    assert nxt == 2
    resumed.run(nxt)
    assert torch.equal(resumed.bank.theta, full.bank.theta)


def test_facade_keys_the_residual_by_client_index():
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    args = _sea(compression="eftopk", topk_ratio=0.2, client_num_in_total=6, client_num_per_round=2)
    M, W = 2, 2
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, W, "cpu", [model] * M, 2, args)
    P = agg.bank.P
    assert agg.ef_res.shape == (6, M, P) and agg.bank.ef_res is agg.ef_res
    g = torch.Generator().manual_seed(3)
    agg.bank.theta.copy_(torch.randn(M, P, generator=g))
    want_res = torch.zeros(6, M, P)
    for rnd in range(3):
        idx = [int(c) for c in agg.sample_round_clients(rnd, 6, 2)]
        theta0 = agg.bank.theta.clone()
        raw = theta0[None] + 0.2 * torch.randn(W, M, P, generator=g)
        for w in range(W):
            sds = {m: ({k: v.clone() for k, v in mutils.unflatten_to_state_dict(raw[w, m], agg.bank.spec).items()},
                       0 if m == M - 1 else 5) for m in range(M)}   # the last slot gets no weight: untouched
            agg.add_local_trained_result(w, sds)
        assert agg.check_whether_all_receive()
        for w, c in enumerate(idx):
            up = raw[w:w + 1].clone()
            n = torch.ones(1, M)
            n[0, -1] = 0
            ref.eftopk_slots_(up, theta0, want_res[c:c + 1], n, agg.topk_k)
            assert torch.equal(agg.upload[w, :-1], up[0, :-1]), (rnd, w)
        assert torch.equal(agg.ef_res, want_res), rnd
        agg._aggregate_models()
    assert bool((want_res != 0).any()) and bool((want_res[:, -1] == 0).all())
    plain = _BaseAggregator(None, None, None, None, None, None, None, W, "cpu", [model] * M, 2, _sea())
    assert plain.topk_k == 0 and plain.ef_res is None


def test_facade_inproc_runs_with_eftopk():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args, run_facade
    from feddrift_b200.utils.metrics import set_sink
    base = ["--engine", "facade", "--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60"]
    p = add_args(argparse.ArgumentParser())
    se, sn = MetricsSink(), MetricsSink()
    e = run_facade(p.parse_args(base + ["--compression", "eftopk", "--topk_ratio", "0.2"]), set_sink(se))
    run_facade(p.parse_args(base), set_sink(sn))
    assert len(e["history"]) == 2 and all(0 <= h["test_acc"] <= 1 for h in e["history"])
    assert se.series("Train/Loss") != sn.series("Train/Loss")


@pytest.mark.parametrize("kw", [dict(compression="eftopk", topk_ratio=0.0), dict(compression="eftopk", topk_ratio=1.5),
                                dict(compression="none", topk_ratio=-1.0), dict(compression="qsgd", topk_ratio=float("nan")),
                                dict(compression="eftopk", topk_ratio=float("inf"))])
def test_rejections(kw):
    with pytest.raises(ValueError):
        DriftSim(_sea(**kw), device="cpu", sink=MetricsSink())
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    with pytest.raises(ValueError):
        _BaseAggregator(None, None, None, None, None, None, None, 2, "cpu", [mutils.create_model("fnn", 2, 3)], 2, _sea(**kw))
    st = dict(make_state(C=8, S=20), **kw)
    with pytest.raises(ValueError):
        ref.fed_round_small(st, 1)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert a.topk_ratio == 0.01 and make_args().topk_ratio == 0.01
    a = p.parse_args(["--compression", "eftopk", "--topk_ratio", "0.05"])
    assert (a.compression, a.topk_ratio) == ("eftopk", 0.05)
    with pytest.raises(SystemExit):
        p.parse_args(["--compression", "topk"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2e_sea_fnn_100clients_eftopk_feddrift"]
    assert (cfg["compression"], cfg["topk_ratio"]) == ("eftopk", 0.25)
