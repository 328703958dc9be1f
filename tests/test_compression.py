"""QSGD upload compression (``--compression qsgd``) of the continual engines on the CPU: the quantizer's definition (levels,
pass-through entries, unbiasedness, draws), the accounting formula, the round oracle, the device engine's two routes, the
raw-update hooks, the façade, checkpoint resume and the rejected configurations."""
import argparse
import copy
import math

import pytest
import torch

from feddrift_b200.models import utils as mutils
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, checkpoint, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state
from test_robust_defense import _BnNet, _weights


def _arena(C=3, M=2, P=37, pad=5, scale=0.3, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(M, P + pad, generator=g)   # a padded bank row
    rows = theta[None, :, :P] + scale * torch.randn(C, M, P, generator=g)
    return rows, theta


def _levels(rows, before, theta, s, b, mask=None):
    """(q, a) per entry from the definition: the level the quantizer picked and the scaled magnitude it started from."""
    C, M, P = rows.shape
    d = before - theta[None, :, :P]
    ad = d.abs() if mask is None else torch.where(mask, d.abs(), torch.zeros_like(d))
    nb = math.ceil(P / b)
    sig = torch.nn.functional.pad(ad, (0, nb * b - P)).view(C, M, nb, b).amax(3).repeat_interleave(b, 2)[..., :P]
    a = (ad / sig) * s
    q = ((rows - theta[None, :, :P]).abs() / sig * s).round()
    return q, a, sig


@pytest.mark.parametrize("s,b", [(1, 5), (4, 8), (16, 512), (7, 1), (3, 37)])
def test_every_quantized_entry_is_a_level(s, b):
    rows, theta = _arena()
    before = rows.clone()
    ref.qsgd_slots_(rows, theta, None, s, b, None, seed=11)
    q, a, sig = _levels(rows, before, theta, s, b)
    d = before - theta[None, :, :37]
    want = theta[None, :, :37] + torch.copysign(sig * (q / s), d)
    on = sig > 0
    assert torch.equal(rows[on], want[on])
    assert bool(((q >= 0) & (q <= s)).all())
    fl = torch.floor(a)
    assert bool(((q == fl) | (q == fl + 1))[on].all())
    if s == 1:   # ternary: every entry is θ or θ ± σ_k
        tern = torch.stack([theta[None, :, :37] + sig, theta[None, :, :37] - sig, theta[None, :, :37].expand_as(sig)])
        assert bool((rows[None] == tern).any(0)[on].all())


def test_masked_entries_skipped_rows_and_zero_buckets_are_untouched():
    rows, theta = _arena(C=3, M=2, P=40)
    rows[0, 1, 8:16] = theta[1, 8:16]   # bucket 1 of row (0, 1) has no update: σ == 0
    before = rows.clone()
    n = torch.ones(3, 2)
    n[2, 0] = 0
    mask = torch.ones(40, dtype=torch.bool)
    mask[::3] = False
    ref.qsgd_slots_(rows, theta, n, 4, 8, mask, seed=5)
    assert torch.equal(rows[..., ~mask], before[..., ~mask])
    assert torch.equal(rows[2, 0], before[2, 0])
    assert torch.equal(rows[0, 1, 8:16], before[0, 1, 8:16])
    assert not torch.equal(rows[0, 0], before[0, 0])
    # the scales come from the trainable entries only: a huge masked entry changes nothing
    r2, _ = _arena(C=3, M=2, P=40)
    r2[0, 1, 8:16] = theta[1, 8:16]
    r2[..., 0] = 1e6
    ref.qsgd_slots_(r2, theta, n, 4, 8, mask, seed=5)
    assert torch.equal(r2[..., mask], rows[..., mask])


def test_unbiased_over_seeds():
    rows, theta = _arena(C=1, M=1, P=64, scale=1.0)
    S, N = 2, 4000
    acc = torch.zeros(64, dtype=torch.float64)
    acc2 = torch.zeros(64, dtype=torch.float64)
    for k in range(N):
        r = rows.clone()
        ref.qsgd_slots_(r, theta, None, S, 16, None, seed=ref.compress_seed(7, k))
        v = r[0, 0].double()
        acc += v
        acc2 += v * v
    mean = acc / N
    sd = (acc2 / N - mean * mean).clamp(min=0).sqrt()
    # per entry |mean − raw| ≤ 5 standard errors (a Bernoulli draw between two adjacent levels; the sample sd bounds it)
    err = (mean - rows[0, 0].double()).abs()
    bound = 5 * sd / math.sqrt(N) + 1e-6
    assert bool((err <= bound).all()), (err / bound).max()


def test_draws_depend_on_seed_and_round_only():
    rows, theta = _arena()
    a, b, c = rows.clone(), rows.clone(), rows.clone()
    ref.qsgd_slots_(a, theta, None, 2, 8, None, ref.compress_seed(99, 3))
    ref.qsgd_slots_(b, theta, None, 2, 8, None, ref.compress_seed(99, 3))
    ref.qsgd_slots_(c, theta, None, 2, 8, None, ref.compress_seed(99, 4))
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert ref.compress_seed(99, 3) != ref.defense_seed(99, 3)
    assert len({ref.compress_seed(1234, r) for r in range(50)} | {ref.compress_seed(1235, 0)}) == 51
    u = ref.uniform_hash(77, [4, 1], 10)
    assert u.dtype == torch.float32 and bool(((u >= 0) & (u < 1)).all())
    assert torch.equal(u, ref.uniform_hash(77, range(5), 10)[[4, 1]])


def test_upload_bits_formula():
    assert ref.qsgd_upload_bits(1000, 0, 16, 512) == 32 * 2 + 6 * 1000
    assert ref.qsgd_upload_bits(1000, 24, 1, 100) == 32 * 10 + 2 * 1000 + 32 * 24
    assert ref.qsgd_upload_bits(10, 0, 65535, 1) == 32 * 10 + 17 * 10
    assert ref.qsgd_upload_bits(10, 0, 15, 1000) == 32 + 5 * 10
    mask = torch.tensor([True] * 4 + [False] * 8 + [True] * 4)   # buckets of 4: 0 and 3 hold trainable entries
    assert ref.qsgd_upload_bits(8, 8, 4, 4, mask) == 32 * 2 + 4 * 8 + 32 * 8


@pytest.mark.parametrize("kw", [dict(compression="topk"), dict(compression="qsgd", quantize_level=0),
                                dict(compression="qsgd", quantize_level=65536), dict(compression="qsgd", quantize_level=2.5),
                                dict(compression="qsgd", quantize_bucket=0), dict(compression="none", quantize_bucket=-3),
                                dict(compression="qsgd", quantize_level=float("nan"))])
def test_rejections(kw):
    with pytest.raises(ValueError):
        DriftSim(_sea(**kw), device="cpu", sink=MetricsSink())
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    with pytest.raises(ValueError):
        _BaseAggregator(None, None, None, None, None, None, None, 2, "cpu", [mutils.create_model("fnn", 2, 3)], 2, _sea(**kw))
    st = dict(make_state(C=8, S=20), compression=kw["compression"], quantize_level=kw.get("quantize_level", 16),
              quantize_bucket=kw.get("quantize_bucket", 512))
    with pytest.raises(ValueError):
        ref.fed_round_small(st, 1)


def _with_q(st, s=2, b=16):
    return dict(st, compression="qsgd", quantize_level=s, quantize_bucket=b)


def test_oracle_round_is_the_average_of_quantized_uploads():
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    plain = copy.deepcopy(st)
    plain["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(plain, 1)
    q = _with_q(copy.deepcopy(st))
    q["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(q, 1)
    n = _weights(st)
    want_up = plain["client_out"].clone()
    ref.qsgd_slots_(want_up, theta0, n, 2, 16, None, ref.compress_seed(st["seed"], 0))
    assert torch.equal(q["client_out"], want_up)   # the export holds the uploads as quantized
    assert not torch.equal(want_up, plain["client_out"])
    want = theta0.clone()
    for m in range(M):
        tot = n[:, m].double().sum()
        if tot > 0:
            want[m] = sum(want_up[c, m] * (float(n[c, m]) / float(tot)) for c in range(C) if n[c, m] > 0)
    assert torch.allclose(q["theta"], want, rtol=0, atol=1e-6)
    for k in ("opt_m", "opt_step"):   # local training does not see the quantization
        assert torch.equal(q[k], plain[k]), k


def test_oracle_quantizes_before_the_defense():
    st = make_state(C=8, S=40, epochs=2)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    q = _with_q(copy.deepcopy(st))
    q["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(q, 1)
    qd = dict(_with_q(copy.deepcopy(st)), defense="weak_dp", norm_bound=0.1, stddev=0.01)
    ref.fed_round_small(qd, 1)
    n = _weights(st)
    up = q["client_out"].clone()
    ref.robust_clip_slots_(up, theta0, n, 0.1, None, 0.01, ref.defense_seed(st["seed"], 0))
    want = theta0.clone()
    ref.cluster_aggregate_(want, up, n)
    assert torch.allclose(qd["theta"], want, rtol=0, atol=1e-6)


def _sea(**kw):
    d = dict(client_num_in_total=8, comm_round=3, total_train_iteration=3, sample_num=40, epochs=2)
    d.update(kw)
    return make_args(**d)


def _run(args, end=None):
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    out = sim.run(end_iteration=end)
    return sim, out


def test_drift_sim_fused_and_generic_routes_agree_and_log_the_upload_size():
    args = _sea(compression="qsgd", quantize_level=2, quantize_bucket=8)
    fused, out = _run(args, end=2)
    generic = DriftSim(copy.deepcopy(args), device="cpu", sink=MetricsSink())
    generic.algo.fused_ok = lambda: False
    generic.run(end_iteration=2)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    plain, _ = _run(_sea(), end=2)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, plain.bank.theta)
    bits = fused.sink.series("Comm/UploadBits")
    P = fused.bank.P
    assert bits == [ref.qsgd_upload_bits(P, 0, 2, 8)] * 2
    assert fused.sink.series("Comm/CompressionRatio") == [32.0 * P / bits[0]] * 2
    assert not plain.sink.series("Comm/UploadBits")


def test_none_is_identical_to_the_default():
    a, oa = _run(_sea(compression="none", quantize_level=3, quantize_bucket=7))
    b, ob = _run(_sea())
    assert torch.equal(a.bank.theta, b.bank.theta) and oa["history"] == ob["history"]


def _cnn_sim(**kw):
    d = dict(model="cnn", dataset="MNIST", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1", concept_drift_algo_arg="",
             change_points="A", sample_num=8, batch_size=8, comm_round=2, total_train_iteration=2, epochs=1, client_optimizer="sgd",
             lr=0.05)
    d.update(kw)
    sim = DriftSim(make_args(**d), device="cpu", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    return sim


def _record_qsgd(monkeypatch):
    """Wrap ``ops.qsgd_slots_``: records (raw rows, n, quantized rows) of every call."""
    from feddrift_b200 import ops
    calls = []
    real = ops.qsgd_slots_

    def wrapped(rows, theta, n=None, *a, **k):
        raw = rows.clone()
        out = real(rows, theta, n, *a, **k)
        calls.append((raw, None if n is None else n.clone(), rows.clone()))
        return out
    monkeypatch.setattr(ops, "qsgd_slots_", wrapped)
    return calls


@pytest.mark.parametrize("per_round", [4, 2])
def test_generic_cnn_round_aggregates_the_quantized_arena(per_round, monkeypatch):
    sim = _cnn_sim(compression="qsgd", quantize_level=2, quantize_bucket=64, client_num_per_round=per_round)
    assert sim.spec is None
    calls = _record_qsgd(monkeypatch)
    theta0 = sim.bank.theta.clone()
    before = sim.clients.params.clone()
    sim.run_rounds(1)
    raw, n, _ = calls[0]
    want_up = raw.clone()
    ref.qsgd_slots_(want_up, theta0, n, 2, 64, sim.defense_mask, ref.compress_seed(0 * 7919 + 13, 0))
    assert torch.equal(sim.clients.params, want_up)
    sel = n > 0
    assert not torch.equal(want_up[sel], raw[sel])
    if per_round < 4:   # clients that were not sampled neither trained nor were quantized
        idle = ~sel.any(1)
        assert bool(idle.any())
        assert torch.equal(sim.clients.params[idle], before[idle])
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
    before = up.clone()
    ref.qsgd_slots_(up, bank.theta, torch.ones(C, M), 2, 16, wmask, seed=9)
    assert torch.equal(up[..., ~wmask], before[..., ~wmask])
    assert not torch.equal(up[..., wmask], before[..., wmask])


@pytest.mark.parametrize("algo", [("softcluster", "cfl_0.1_win-1"), ("clusterfl", "win-1")])
def test_raw_update_hooks_see_quantized_uploads(algo, monkeypatch):
    args = _sea(concept_drift_algo=algo[0], concept_drift_algo_arg=algo[1], concept_num=2, comm_round=3,
                compression="qsgd", quantize_level=1, quantize_bucket=8)
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    sim.begin_time_step(0)
    calls = _record_qsgd(monkeypatch)
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
    raw, n, quant = calls[0]
    sel = n > 0
    assert torch.equal(seen[0], quant)
    assert not torch.equal(quant[sel], raw[sel])


def test_facade_aggregator_quantizes_each_upload():
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    args = _sea(compression="qsgd", quantize_level=3, quantize_bucket=16, dummy_arg=2, curr_train_iteration=1)
    M, C = 3, 4
    model = mutils.create_model("fnn", 2, 3)
    agg = _BaseAggregator(None, None, None, None, None, None, None, C, "cpu", [model] * M, 2, args)
    P = agg.bank.P
    g = torch.Generator().manual_seed(3)
    agg.bank.theta.copy_(torch.randn(M, P, generator=g))
    seed = 2 * 7919 + 13 + 1000003 * 1
    for rnd in range(2):
        theta0 = agg.bank.theta.clone()
        raw = theta0[None] + 0.2 * torch.randn(C, M, P, generator=g)
        for w in range(C):
            sds = {}
            for m in range(M):
                sd = {k: v.clone() for k, v in mutils.unflatten_to_state_dict(raw[w, m], agg.bank.spec).items()}
                sds[m] = (sd, 0 if m == M - 1 else 5)   # the last slot gets no weight: not quantized
            agg.add_local_trained_result(w, sds)
        assert agg.check_whether_all_receive()
        want = raw.clone()
        n = torch.ones(C, M)
        n[:, -1] = 0
        ref.qsgd_slots_(want, theta0, n, 3, 16, None, ref.compress_seed(seed, rnd))
        assert torch.equal(agg.upload[:, :-1], want[:, :-1]), rnd
        assert not torch.equal(agg.upload[:, :-1], raw[:, :-1])
        agg._aggregate_models()
    plain = _BaseAggregator(None, None, None, None, None, None, None, C, "cpu", [model] * M, 2, _sea())
    assert plain.q_level == 0


def test_facade_inproc_runs_with_qsgd():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args, run_facade
    from feddrift_b200.utils.metrics import set_sink
    base = ["--engine", "facade", "--comm_round", "3", "--total_train_iteration", "2", "--sample_num", "60"]
    p = add_args(argparse.ArgumentParser())
    sq, sn = MetricsSink(), MetricsSink()
    q = run_facade(p.parse_args(base + ["--compression", "qsgd", "--quantize_level", "1", "--quantize_bucket", "4"]), set_sink(sq))
    run_facade(p.parse_args(base), set_sink(sn))
    assert len(q["history"]) == 2 and all(0 <= h["test_acc"] <= 1 for h in q["history"])
    assert sq.series("Train/Loss") != sn.series("Train/Loss")


def test_checkpoint_resume_with_qsgd(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, compression="qsgd", quantize_level=2, quantize_bucket=8)
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    full.run()
    part = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    part.run(0, 2)
    resumed = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    nxt = checkpoint.resume(resumed, checkpoint.latest(str(tmp_path)))
    assert nxt == 2
    resumed.run(nxt)
    assert torch.equal(resumed.bank.theta, full.bank.theta)


def test_cli_flags_and_config():
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    a = p.parse_args([])
    assert (a.compression, a.quantize_level, a.quantize_bucket) == ("none", 16, 512)
    with pytest.raises(SystemExit):
        p.parse_args(["--compression", "topk"])
    from feddrift_b200.experiments.configs import CONFIGS
    cfg = CONFIGS["cfg2q_sea_fnn_100clients_qsgd_feddrift"]
    assert (cfg["compression"], cfg["quantize_level"]) == ("qsgd", 4)
