"""Centered-clipping cluster aggregation (``--aggregation_rule centered_clip``) of the continual engines on the CPU: the oracle
against an independent numpy float32 definition, the parameters, the mean and norm-clipping special cases, the attacker
bound, the per-slot state's lifetime, the device engine's two routes, the façade, the CLI, the config and the Byzantine
scenario."""
import argparse
import copy

import numpy as np
import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state
from test_robust_agg import BYZ, BYZ_KW, _same
from test_robust_defense import _weights

f32 = np.float32


def np_cclip(theta, uploads, n, center, tau, iters, mask=None):
    """Independent definition in numpy, every float32 operation rounded on its own: d = x − θ, v = h; L times u = d − v,
    r² = Σ mask·u² in float64, s = fl32(min(1, fl32(τ) / r)), v = v + (Σ_{s ≠ 0} s·u in client order) / n; θ ← θ + v,
    h ← v; a NaN distance makes θ_m and h_m NaN.  Returns (θ, h) as new tensors."""
    th = theta.numpy().copy()
    h = center.numpy().copy()
    X = uploads.numpy()
    C, M, P = X.shape
    keep = np.ones(P, bool) if mask is None else mask.numpy().astype(bool)
    tau_d = float(f32(tau))
    for m in range(M):
        rows = [c for c in range(C) if float(n[c, m]) > 0]
        if not rows:
            continue
        t0 = th[m, :P].astype(f32)
        d = [(X[c, m].astype(f32) - t0).astype(f32) for c in rows]
        v = h[m].astype(f32).copy()
        nan = False
        for _ in range(iters):
            u = [(di - v).astype(f32) for di in d]
            with np.errstate(invalid="ignore", over="ignore"):
                r2 = [float(np.sum(np.where(keep, ui.astype(np.float64) ** 2, 0.0))) for ui in u]
            if any(np.isnan(r) for r in r2):
                nan = True
                break
            with np.errstate(divide="ignore"):
                s = [f32(min(1.0, tau_d / np.sqrt(np.float64(r)))) for r in r2]
            acc = np.zeros(P, f32)
            for si, ui in zip(s, u):
                if si != 0:
                    acc = (acc + (si * ui).astype(f32)).astype(f32)
            v = (v + (acc / f32(len(rows))).astype(f32)).astype(f32)
        if nan:
            th[m, :P] = np.nan
            h[m] = np.nan
        else:
            th[m, :P] = (t0 + v).astype(f32)
            h[m] = v
    return torch.from_numpy(th), torch.from_numpy(h)


def _arena(C, M=4, P=13, pad=0, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, P + pad, generator=g)
    ups = bank[None, :, :P] + scale * torch.randn(C, M, P, generator=g)
    n = (torch.rand(C, M, generator=g) * 5).floor() + (torch.arange(C) % 2)[:, None]
    center = 0.3 * torch.randn(M, P, generator=g)
    return bank, ups, n, center


# ----------------------------------------------------------------------------- parameters
def test_cclip_params():
    assert ref.cclip_params(1.0, 1) == (1.0, 1)
    assert ref.cclip_params(0.25, 100) == (0.25, 100)
    assert ref.cclip_params("2.5", np.int64(3)) == (2.5, 3)
    for tau in (0.0, -1.0, float("nan"), float("inf"), -float("inf"), 1e-46, 1e39, True, None, "x"):
        with pytest.raises(ValueError, match="cclip_tau"):
            ref.cclip_params(tau, 1)
    for it in (0, 101, -1, True, False, 1.0, 2.5, "3", None):
        with pytest.raises(ValueError, match="cclip_iters"):
            ref.cclip_params(1.0, it)
    assert "centered_clip" in ref.AGGREGATION_RULES and ref.aggregation_params("centered_clip", 0.1) == ("centered_clip", 0.1)


@pytest.mark.parametrize("kw", [dict(cclip_tau=0.0), dict(cclip_tau=float("nan")), dict(cclip_tau=1e39), dict(cclip_iters=0),
                                dict(cclip_iters=101), dict(cclip_iters=True), dict(aggregation_rule="mean", cclip_tau=-2.0),
                                dict(aggregation_rule="median", cclip_iters=2.0)])
def test_rejections(kw):
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    from feddrift_b200.models import utils as mutils
    kw = dict(dict(aggregation_rule="centered_clip"), **kw)
    with pytest.raises(ValueError):
        DriftSim(_sea(**kw), device="cpu", sink=MetricsSink())
    with pytest.raises(ValueError):
        _BaseAggregator(None, None, None, None, None, None, None, 2, "cpu", [mutils.create_model("fnn", 2, 3)], 2, _sea(**kw))
    with pytest.raises(ValueError):
        ref.fed_round_small(dict(make_state(C=8, S=20), **kw), 1)


# ----------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("iters", [1, 2, 5])
@pytest.mark.parametrize("C", [1, 2, 3, 9])
@pytest.mark.parametrize("masked", [False, True])
def test_oracle_matches_numpy(iters, C, masked):
    bank, ups, n, center = _arena(C, pad=3, seed=C * 10 + iters)
    n[:, 1] = 0                                            # a slot without participants keeps θ and h
    if C >= 2:
        n[:, 2] = 0
        n[0, 2] = 1                                         # n = 1
    mask = None
    if masked:
        mask = torch.ones(13, dtype=torch.bool)
        mask[[2, 7]] = False
    for tau in (0.05, 0.7, 1e6):
        th, h = bank.clone(), center.clone()
        counts = ref.cclip_aggregate_slots_(th, ups, n, h, tau, iters, mask)
        want_th, want_h = np_cclip(bank, ups, n, center, tau, iters, mask)
        assert _same(th, want_th) and _same(h, want_h), (tau, iters, C)
        assert torch.equal(counts, (n > 0).sum(0).float())
        assert torch.equal(th[:, 13:], bank[:, 13:])        # padding untouched
        assert torch.equal(th[1], bank[1]) and torch.equal(h[1], center[1])


def test_infinite_row_is_dropped_and_nan_row_poisons_the_slot():
    bank, ups, n, center = _arena(6, seed=5)
    n[:] = 1
    ups[2, 0, 4] = float("inf")                             # slot 0: r = +∞, s = 0, the row is left out
    ups[3, 1, 6] = float("nan")                             # slot 1: a NaN distance
    mask = torch.ones(13, dtype=torch.bool)
    mask[9] = False
    ups[4, 2, 9] = float("nan")                             # slot 2: NaN outside the mask reaches v through s·u
    for iters in (1, 3):
        th, h = bank.clone(), center.clone()
        ref.cclip_aggregate_slots_(th, ups, n, h, 0.5, iters, mask)
        want_th, want_h = np_cclip(bank, ups, n, center, 0.5, iters, mask)
        assert _same(th, want_th) and _same(h, want_h)
        assert torch.isfinite(th[0]).all() and torch.isfinite(h[0]).all()
        assert (th[1].view(torch.int32) == 0x7FC00000).all() and (h[1].view(torch.int32) == 0x7FC00000).all()
        assert torch.isnan(th[2, 9]) and torch.isfinite(th[3]).all()
        # the +∞ row contributes nothing but still counts in n
        rest = ups[[0, 1, 3, 4, 5], 0:1].clone()
        th2, h2 = bank[0:1].clone(), center[0:1].clone()
        ref.cclip_aggregate_slots_(th2, rest, torch.ones(5, 1), h2, 0.5, 1, mask)
        if iters == 1:
            v5 = h2[0] - center[0]
            assert torch.allclose(h[0] - center[0], v5 * 5 / 6, rtol=1e-5, atol=1e-6)


def test_many_clients_and_a_padded_bank():
    bank, ups, n, center = _arena(40, M=2, P=21, pad=11, seed=8, scale=0.5)
    th, h = bank.clone(), center.clone()
    ref.cclip_aggregate_slots_(th, ups, n, h, 0.8, 3)
    want_th, want_h = np_cclip(bank, ups, n, center, 0.8, 3)
    assert _same(th, want_th) and _same(h, want_h)


# ----------------------------------------------------------------------------- properties
def _ulps(a, b):
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return (ia - ib).abs()


def test_large_radius_is_the_unweighted_mean():
    """τ above every distance, h = 0, L = 1: every s = 1 and θ + v is the unweighted mean of the uploads (each counted once,
    the weights ignored), to 1 ulp of the correctly rounded mean."""
    g = torch.Generator().manual_seed(2)
    M, P, C = 3, 17, 7
    bank = 1.0 + torch.rand(M, P, generator=g)
    ups = bank[None] + 0.01 * torch.randn(C, M, P, generator=g)
    n = (torch.rand(C, M, generator=g) * 9).floor() + 1
    th, h = bank.clone(), torch.zeros(M, P)
    ref.cclip_aggregate_slots_(th, ups, n, h, 1e30, 1)
    want = ups.double().mean(0).float()
    assert int(_ulps(th, want).max()) <= 1
    assert torch.equal(h, th - bank) or torch.allclose(h, th - bank, atol=1e-6)


def test_first_round_is_norm_clipping_plus_the_unweighted_mean():
    """h = 0, L = 1: centered clipping is K10's norm-difference clipping at bound τ around θ followed by the unweighted mean."""
    for seed in range(3):
        bank, ups, n, _ = _arena(8, seed=seed, scale=0.6)
        tau = 1.2
        th, h = bank.clone(), torch.zeros_like(bank)
        ref.cclip_aggregate_slots_(th, ups, n, h, tau, 1)
        clipped = ups.clone()
        ref.robust_clip_slots_(clipped, bank, n, tau)
        for m in range(bank.shape[0]):
            rows = (n[:, m] > 0).nonzero().flatten()
            if len(rows) == 0:
                assert torch.equal(th[m], bank[m])
                continue
            want = clipped[rows, m].double().mean(0)
            assert torch.allclose(th[m].double(), want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("kind", ["huge", "inf_norm", "aligned"])
def test_attackers_move_one_iteration_by_at_most_a_tau_over_n(kind):
    """Every honest update within τ of v⁰ keeps s = 1, and every attacker's clipped update has norm ≤ τ, so one iteration
    moves v by the honest updates' sum over n plus at most a·τ/n whatever the a attackers send (the attackers' share of
    the denominator costs at most another a·τ/n against the honest mean itself)."""
    g = torch.Generator().manual_seed(11)
    P, honest, a, tau = 29, 9, 3, 0.5
    mask = torch.ones(P, dtype=torch.bool)
    mask[[0, 5]] = False
    theta = torch.randn(1, P, generator=g)
    v0 = 0.2 * torch.randn(1, P, generator=g)
    dirs = torch.randn(honest, P, generator=g)
    dirs = dirs / dirs.norm(dim=1, keepdim=True) * 0.9 * tau * torch.rand(honest, 1, generator=g)
    hon = theta + v0 + dirs
    hon[:, ~mask] = theta[:, ~mask] + v0[:, ~mask]             # masked-out entries carry no update
    if kind == "huge":
        att = theta + 1e6 * torch.randn(a, P, generator=g)
    elif kind == "inf_norm":
        att = theta + 3e18 * torch.ones(a, P)
    else:
        att = theta + v0 + 40.0 * dirs[:1].expand(a, P)
    att[:, ~mask] = theta[:, ~mask] + v0[:, ~mask]
    ups = torch.cat([att, hon])[:, None, :]
    n = torch.ones(honest + a, 1)
    th, h = theta.clone(), v0.clone()
    ref.cclip_aggregate_slots_(th, ups, n, h, tau, 1, mask)
    u = (hon - theta - v0).double()
    ntot = honest + a
    got = h.double()[0]
    near = v0.double()[0] + u.sum(0) / ntot
    far = v0.double()[0] + u.mean(0)
    eps = 1e-5
    assert float((got - near)[mask].norm()) <= a * tau / ntot + eps
    assert float((got - far)[mask].norm()) <= 2 * a * tau / ntot + eps


# ----------------------------------------------------------------------------- ops, server optimizer, fused oracle
def test_ops_dispatch_and_server_optimizer_on_cpu():
    bank, ups, n, center = _arena(6, seed=4)
    th, h = bank.clone(), center.clone()
    counts = ops.cluster_aggregate_(th, ups, n, None, ("centered_clip", 0.1, 0.7, 2), center=h)
    want_th, want_h = np_cclip(bank, ups, n, center, 0.7, 2)
    assert _same(th, want_th) and _same(h, want_h) and torch.equal(counts, (n > 0).sum(0).float())
    with pytest.raises(ValueError, match="center"):
        ops.cluster_aggregate_(bank.clone(), ups, n, None, ("centered_clip", 0.1, 0.7, 2))
    # the center is ignored by the other rules
    a, b = bank.clone(), bank.clone()
    ops.cluster_aggregate_(a, ups, n, None, ("median", 0.1), center=center.clone())
    ops.cluster_aggregate_(b, ups, n, None, ("median", 0.1))
    assert _same(a, b)
    from feddrift_b200.ops.server_opt import SlotServerOpt
    so = SlotServerOpt("adam", bank.shape[0], 13, "cpu", lr=0.05)
    th, h = bank[:, :13].clone(), center.clone()
    ops.cluster_aggregate_(th, ups, n, so, ("centered_clip", 0.1, 0.7, 2), center=h)
    avg, h2 = np_cclip(bank[:, :13].clone(), ups, n, center, 0.7, 2)
    want = bank[:, :13].clone()
    s0, s1, stp = torch.zeros(4, 13), torch.zeros(4, 13), torch.zeros(4, dtype=torch.int32)
    ref.server_opt_slots_(want, avg, (n > 0).any(0), "adam", s0, s1, stp, 0.05)
    assert torch.equal(th, want) and _same(h, h2)


def test_oracle_round_clips_after_compression_attack_and_defense():
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    n = _weights(st)
    att = torch.zeros(C, dtype=torch.bool)
    att[[1, 6]] = True
    kw = dict(compression="qsgd", quantize_level=4, quantize_bucket=8, defense="norm_diff_clipping", norm_bound=0.5,
              attack_type="sign_flip", attack_clients=2, attack_scale=3.0, attackers=att)
    plain = dict(copy.deepcopy(st), **kw)
    plain["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(plain, 1)
    h0 = 0.01 * torch.randn(M, P, generator=torch.Generator().manual_seed(1))
    r = dict(copy.deepcopy(st), aggregation_rule="centered_clip", cclip_tau=0.05, cclip_iters=2, cclip_center=h0.clone(), **kw)
    ref.fed_round_small(r, 1)
    up = plain["client_out"].clone()                              # compressed and attacked
    ref.robust_clip_slots_(up, theta0, n, 0.5, None, 0.0, 0)
    want, want_h = np_cclip(theta0, up, n, h0, 0.05, 2)
    assert _same(r["theta"], want) and _same(r["cclip_center"], want_h)
    fresh = dict(copy.deepcopy(st), aggregation_rule="centered_clip")
    ref.fed_round_small(fresh, 1)                                 # the state is created zero when missing
    assert fresh["cclip_center"].shape == (M, P) and bool(fresh["cclip_center"].any())


def test_oracle_round_state_persists_across_launches():
    st = dict(make_state(C=6, S=30, epochs=2), aggregation_rule="centered_clip", cclip_tau=0.02, cclip_iters=2)
    one, three = copy.deepcopy(st), copy.deepcopy(st)
    m1 = ref.fed_round_small(one, 3)["metrics"]
    m3 = torch.cat([ref.fed_round_small(three, 1)["metrics"] for _ in range(3)])
    assert torch.equal(m1, m3) and _same(one["theta"], three["theta"]) and _same(one["cclip_center"], three["cclip_center"])
    # a slot nobody trains keeps its center
    idle = int((~(st["W"][st["t_cur"]] != 0).any(dim=1)).nonzero()[0])
    h0 = torch.full((st["theta"].shape[0], st["theta"].shape[1]), 0.125)
    r = dict(copy.deepcopy(st), cclip_center=h0.clone())
    ref.fed_round_small(r, 2)
    assert torch.equal(r["cclip_center"][idle], h0[idle]) and not torch.equal(r["cclip_center"], h0)


# ----------------------------------------------------------------------------- the device engine
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


def test_drift_sim_state_lifetime():
    sim = DriftSim(_sea(aggregation_rule="centered_clip", cclip_tau=0.05, cclip_iters=2), device="cpu", sink=MetricsSink())
    assert sim.agg_rule == ("centered_clip", 0.1, 0.05, 2)
    assert sim.bank.cclip_center.shape == (sim.M, sim.bank.P) and not bool(sim.bank.cclip_center.any())
    sim.begin_time_step(0)
    sim.run_rounds(2)
    h = sim.bank.cclip_center.clone()
    assert bool(h.any())
    sim.run_rounds(1)                                             # carried into the next launch
    assert not torch.equal(sim.bank.cclip_center, h)
    sim.end_time_step()
    sim.bank.cclip_center.fill_(0.5)
    sim.bank.reinit(1)
    assert not bool(sim.bank.cclip_center[1].any()) and bool((sim.bank.cclip_center[0] == 0.5).all())
    sim.bank.copy(2, 0)
    assert not bool(sim.bank.cclip_center[2].any()) and bool((sim.bank.cclip_center[0] == 0.5).all())
    sim.bank.copy(0, 0)                                           # a copy onto itself changes nothing
    assert bool((sim.bank.cclip_center[0] == 0.5).all())
    sim.begin_time_step(1)
    assert not bool(sim.bank.cclip_center.any())
    assert DriftSim(_sea(), device="cpu", sink=MetricsSink()).bank.cclip_center is None


def test_drift_sim_fused_and_generic_routes_agree():
    args = _sea(aggregation_rule="centered_clip", cclip_tau=0.05, cclip_iters=2, comm_round=4)
    fused, _ = _run(args, end=2)
    generic, _ = _run(copy.deepcopy(args), end=2, generic=True)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    assert torch.allclose(generic.bank.cclip_center, fused.bank.cclip_center, rtol=1e-4, atol=1e-5)
    plain, _ = _run(_sea(comm_round=4), end=2)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, plain.bank.theta)
    # rounds per launch do not change what the state carries
    split, _ = _run(_sea(aggregation_rule="centered_clip", cclip_tau=0.05, cclip_iters=2, comm_round=4, rounds_per_launch=1), end=2)
    assert _same(split.bank.theta, fused.bank.theta) and _same(split.bank.cclip_center, fused.bank.cclip_center)
    # the flags are ignored by the other rules
    assert _same(_run(_sea(comm_round=4, cclip_tau=3.0, cclip_iters=7), end=2)[0].bank.theta, plain.bank.theta)


def test_checkpoint_resume_needs_no_center(tmp_path):
    """Checkpoints are written at time-step ends, where the center is about to be zeroed: a resumed run is the full one."""
    from feddrift_b200.sim import checkpoint
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=5, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, aggregation_rule="centered_clip", cclip_tau=0.1, cclip_iters=2)
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    full.run()
    part = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    part.run(0, 2)
    resumed = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    nxt = checkpoint.resume(resumed, checkpoint.latest(str(tmp_path)))
    assert nxt == 2
    resumed.run(nxt)
    assert torch.equal(resumed.bank.theta, full.bank.theta) and torch.equal(resumed.bank.cclip_center, full.bank.cclip_center)


def test_facade_aggregator_uses_the_rule():
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    from feddrift_b200.models import utils as mutils
    M, W = 2, 5
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, W, "cpu", [model] * M, 2,
                          _sea(aggregation_rule="centered_clip", cclip_tau=0.4, cclip_iters=3, client_num_in_total=W))
    P = agg.bank.P
    assert agg.bank.cclip_center.shape == (M, P) and not bool(agg.bank.cclip_center.any())
    g = torch.Generator().manual_seed(3)
    agg.bank.theta.copy_(torch.randn(M, P, generator=g))
    h0 = torch.zeros(M, P)
    for rnd in range(2):
        theta0 = agg.bank.theta.clone()
        raw = theta0[None] + torch.randn(W, M, P, generator=g)
        for w in range(W):
            sds = {m: ({k: v.clone() for k, v in mutils.unflatten_to_state_dict(raw[w, m], agg.bank.spec).items()},
                       0 if (m == 1 and w == 0) else 3 + w) for m in range(M)}
            agg.add_local_trained_result(w, sds)
        assert agg.check_whether_all_receive()
        agg._aggregate_models()
        want, h0 = np_cclip(theta0, raw, agg.upload_n.clone(), h0, 0.4, 3)
        assert _same(agg.bank.theta, want) and _same(agg.bank.cclip_center, h0)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.cclip_tau, a.cclip_iters) == (1.0, 1)
    assert (make_args().cclip_tau, make_args().cclip_iters) == (1.0, 1)
    a = p.parse_args(["--aggregation_rule", "centered_clip", "--cclip_tau", "0.25", "--cclip_iters", "3"])
    assert (a.aggregation_rule, a.cclip_tau, a.cclip_iters) == ("centered_clip", 0.25, 3)
    with pytest.raises(SystemExit):
        p.parse_args(["--cclip_iters", "1.5"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2c_sea_fnn_100clients_cclip_feddrift"]
    base = CONFIGS["cfg2_sea_fnn_100clients_feddrift"]
    assert cfg["aggregation_rule"] == "centered_clip" and ref.cclip_params(cfg["cclip_tau"], cfg["cclip_iters"])
    assert {k: v for k, v in cfg.items() if k not in ("aggregation_rule", "cclip_tau", "cclip_iters")} == base
    sim = DriftSim(make_args(**dict(cfg, client_num_in_total=8, sample_num=20)), device="cpu", sink=MetricsSink())
    assert sim.agg_rule == ("centered_clip", 0.1, cfg["cclip_tau"], cfg["cclip_iters"])


# ----------------------------------------------------------------------------- Byzantine scenario
# test_robust_agg's federation; the BYZ clients chosen by attacker_clients upload their reversed update scaled by 10
# (sign_flip) or the honest mean's negation scaled by 10 (ipm).  τ = 0.2: the honest update distances of this federation
# have median ≈ 0.15 in a clean run.  Thresholds fixed from the CPU run (honest clients' accuracy after the last round,
# Test/AccHonest): centered clipping ≈ 0.71 under sign_flip and ≈ 0.68 under ipm, the clean weighted mean ≈ 0.70, the
# attacked mean ≈ 0.42 under both, with a margin
CCLIP_KW = dict(cclip_tau=0.2, cclip_iters=1)
CCLIP_MIN, ATTACKED_MEAN_MAX = 0.64, 0.55


def attacked_honest_acc(rule, attack, device="cpu"):
    sim = DriftSim(make_args(aggregation_rule=rule, attack_type=attack, attack_clients=BYZ, attack_scale=10.0, **CCLIP_KW, **BYZ_KW),
                   device=device, sink=MetricsSink())
    sim.run()
    return sim.sink.series("Test/AccHonest")[-1], sim


@pytest.mark.parametrize("attack", ["sign_flip", "ipm"])
def test_centered_clipping_holds_where_the_mean_breaks(attack):
    mean, _ = attacked_honest_acc("mean", attack)
    cc, sim = attacked_honest_acc("centered_clip", attack)
    assert int(sim.attackers.sum()) == BYZ
    assert cc >= CCLIP_MIN, (cc, mean)
    assert mean <= ATTACKED_MEAN_MAX, (cc, mean)
