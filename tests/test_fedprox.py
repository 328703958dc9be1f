"""FedProx local training (``--fedprox_mu``) of the continual engines on the CPU: the round oracle against hand computations
and ``torch.optim.Adam``, composition with client sampling / a server optimizer / weak DP, the device engine's two routes, the
BatchNorm entries, the façade trainer, checkpoint resume and the rejected values."""
import argparse
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from feddrift_b200 import ops
from feddrift_b200.models import utils as mutils
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, checkpoint, make_args
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state

MU = 0.5


def with_prox(st, mu=MU):
    return dict(st, fedprox_mu=mu)


def _exported(st, rounds=1):
    """Run the oracle on a copy of ``st`` and return (state, the local models of the last round [C, M, P])."""
    st = copy.deepcopy(st)
    C, (M, P) = st["X"].shape[1], st["theta"].shape
    st["client_out"] = torch.zeros(C, M, P)
    ref.fed_round_small(st, rounds)
    return st, st["client_out"]


def _batches(st, c, m):
    """The minibatches (x, y) of every local step of pair (c, m) in round 0, as the oracle draws them."""
    T1, C, S = st["X"].shape[:3]
    B, t = int(st["batch_size"]), int(st["t_cur"])
    nb = (st["nsamp"].to(torch.int64) + B - 1) // B
    _, sampler = ref._pair_plan(st, c, m, t, nb, B)
    Xc, Yc = st["X"][:, c].reshape(T1 * S, -1), st["Y"][:, c].reshape(T1 * S)
    out = []
    for e in range(int(st["epochs"])):
        h1 = ref.batch_hash(int(st["seed"]), int(st["round0"]), c, m, e)
        idx = sampler(h1, ref.mix32(h1 ^ 0x68E31DA4))
        out.append((Xc[idx], Yc[idx]))
    return out


def _grad(st, w, x, y):
    return ref.mlp_loss_grad(w, x, y, st["kind"], st["din"], st["hid"], st["dout"])[1]


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_oracle_mu_zero_and_one_step_are_bit_identical(optimizer):
    st = make_state(C=8, S=40, epochs=3, optimizer=optimizer)
    a, ua = _exported(st)
    b, ub = _exported(with_prox(st, 0.0))
    assert torch.equal(a["theta"], b["theta"]) and torch.equal(ua, ub)
    one = make_state(C=8, S=40, epochs=1, optimizer=optimizer)
    a, ua = _exported(one)
    b, ub = _exported(with_prox(one))
    assert torch.equal(a["theta"], b["theta"]) and torch.equal(ua, ub) and torch.equal(a["opt_m"], b["opt_m"])
    c, uc = _exported(with_prox(st))   # three steps: the proximal term acts
    assert not torch.equal(uc, _exported(st)[1])


def test_oracle_sgd_two_steps_with_lr_mu_one():
    st = make_state(C=6, S=40, epochs=2, optimizer="sgd")
    lr = float(st["lr"])
    _, up = _exported(with_prox(st, 1.0 / lr))
    theta = st["theta"]
    c, m = 1, 1
    (x0, y0), (x1, y1) = _batches(st, c, m)
    w1 = theta[m] - lr * _grad(st, theta[m], x0, y0)
    want = theta[m] - lr * _grad(st, w1, x1, y1)   # w1 − lr·(g(w1) + (1/lr)·(w1 − θ_m))
    assert torch.allclose(up[c, m], want, rtol=0, atol=1e-6), (up[c, m] - want).abs().max()


def test_oracle_adam_equals_torch_adam_on_the_proximal_objective():
    st = make_state(C=6, S=40, epochs=5)
    _, up = _exported(with_prox(st))
    theta = st["theta"]
    c, m = 2, 1
    w = theta[m].clone().requires_grad_(True)
    opt = torch.optim.Adam([w], lr=float(st["lr"]), weight_decay=float(st["wd"]), amsgrad=True)
    for x, y in _batches(st, c, m):
        opt.zero_grad()
        logits = ref.mlp_forward(w, x, st["kind"], st["din"], st["hid"], st["dout"])
        loss = F.cross_entropy(logits, y.long()) + MU / 2 * (w - theta[m]).pow(2).sum()
        loss.backward()
        opt.step()
    assert torch.allclose(up[c, m], w.detach(), rtol=0, atol=1e-6), (up[c, m] - w.detach()).abs().max()


def test_composes_with_participation_server_adam_and_weak_dp():
    from test_server_opt import with_server_opt
    st = make_state(C=8, S=40, epochs=3)
    table = torch.zeros(2, 8, dtype=torch.bool)
    table[0, [0, 2, 5, 7]] = True
    st["participation"] = table
    st = with_server_opt(dict(st, defense="weak_dp", norm_bound=0.1, stddev=0.01), "adam")
    a = with_prox(copy.deepcopy(st))
    ref.fed_round_small(a, 1)
    plain = copy.deepcopy(st)
    ref.fed_round_small(plain, 1)
    for c in (1, 3, 4, 6):   # non-participants did not train
        for k in ("opt_m", "opt_v", "opt_vmax", "opt_step"):
            assert torch.equal(a[k][c], st[k][c]), (c, k)
    assert torch.equal(a["theta"][3], st["theta"][3])   # slot 3 has no member: keeps its model and state
    assert a["server_step"].tolist() == plain["server_step"].tolist() == [1, 1, 1, 0]
    assert torch.equal(a["opt_step"], plain["opt_step"])
    assert not torch.allclose(a["theta"], plain["theta"])
    # the defense clips the prox-trained uploads around θ_m: the average equals the one of the defended local models
    b = with_prox(copy.deepcopy(st))
    b.pop("server_opt")
    _, up = _exported(b)
    n = torch.zeros(8, 4)
    trained = up.abs().sum(-1) > 0
    B_, t = int(st["batch_size"]), int(st["t_cur"])
    nb = (st["nsamp"].to(torch.int64) + B_ - 1) // B_
    for c, m in trained.nonzero().tolist():
        n[c, m] = ref._pair_plan(st, c, m, t, nb, B_)[0]
    ref.robust_clip_slots_(up, st["theta"], n, 0.1, None, 0.01, ref.defense_seed(st["seed"], 0))
    want = st["theta"].clone()
    ref.cluster_aggregate_(want, up, n)
    got = copy.deepcopy(b)
    ref.fed_round_small(got, 1)
    assert torch.allclose(got["theta"], want, rtol=0, atol=1e-6)


def test_row_optimizer_references_apply_the_proximal_term():
    g = torch.Generator().manual_seed(4)
    R, P, A = 5, 11, 3
    anchor = torch.randn(A, P + 5, generator=g)   # padded rows
    rows = torch.tensor([2, 0, 1, 2, 0], dtype=torch.int32)
    mask = (torch.rand(P, generator=g) > 0.3).to(torch.uint8)
    p0, grad = torch.randn(R, P, generator=g), torch.randn(R, P, generator=g)
    prox = (MU, anchor, rows, mask)
    want = p0 - 0.1 * (grad + MU * mask * (p0 - anchor[rows.long(), :P]))
    p = p0.clone()
    ops.sgd_rows_(p, grad, 0.1, prox=prox)
    assert torch.allclose(p, want, rtol=0, atol=1e-6)
    rm = torch.tensor([1, 0, 1, 1, 0], dtype=torch.uint8)
    p = p0.clone()
    ops.sgd_rows_(p, grad, 0.1, row_mask=rm, prox=prox)
    assert torch.equal(p[1], p0[1]) and torch.equal(p[4], p0[4]) and torch.allclose(p[0], want[0], rtol=0, atol=1e-6)
    z = lambda: torch.zeros(R, P)   # noqa: E731
    pa, pb = p0.clone(), p0.clone()
    sa, sb = torch.zeros(R, dtype=torch.int32), torch.zeros(R, dtype=torch.int32)
    ma, va, xa, mb, vb, xb = z(), z(), z(), z(), z(), z()
    ops.adam_amsgrad_rows_(pa, grad.clone(), ma, va, xa, sa, 0.01, 1e-3, prox=prox)
    geff = grad + MU * mask * (p0 - anchor[rows.long(), :P])
    ops.adam_amsgrad_rows_(pb, geff, mb, vb, xb, sb, 0.01, 1e-3)
    assert torch.equal(pa, pb) and torch.equal(ma, mb) and torch.equal(sa, sb)


def _sea(**kw):
    d = dict(client_num_in_total=8, comm_round=3, total_train_iteration=3, sample_num=40, epochs=3)
    d.update(kw)
    return make_args(**d)


def _run(args, end=None):
    sim = DriftSim(args, device="cpu", sink=MetricsSink())
    out = sim.run(end_iteration=end)
    return sim, out


def test_drift_sim_fused_and_generic_routes_agree():
    args = _sea(fedprox_mu=MU)
    fused, out = _run(args, end=2)
    assert fused._small is None or fused._small.get("fedprox_mu") == MU
    generic = DriftSim(copy.deepcopy(args), device="cpu", sink=MetricsSink())
    generic.algo.fused_ok = lambda: False
    generic.run(end_iteration=2)
    assert torch.allclose(generic.bank.theta, fused.bank.theta, rtol=1e-4, atol=1e-5)
    plain, _ = _run(_sea(), end=2)
    assert torch.isfinite(fused.bank.theta).all() and not torch.allclose(fused.bank.theta, plain.bank.theta)
    zero, _ = _run(_sea(fedprox_mu=0.0), end=2)
    assert torch.equal(zero.bank.theta, plain.bank.theta)
    assert all(h["test_acc"] == h["test_acc"] for h in out["history"])


def _resnet_round(mu, epochs):
    sim = DriftSim(make_args(model="resnet18", dataset="cifar10", client_num_in_total=2, concept_num=2, concept_drift_algo="win-1",
                             concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=1,
                             total_train_iteration=2, epochs=epochs, client_optimizer="sgd", lr=0.05, fedprox_mu=mu),
                   device="cpu", sink=MetricsSink())
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    sim.run_rounds(1)
    return sim


def test_generic_batchnorm_entries_get_no_proximal_term():
    a, b = _resnet_round(5.0, 2), _resnet_round(0.0, 2)
    wmask = mutils.weight_param_mask(a.bank.spec)[: a.bank.P]
    assert a.prox_mask is not None and not bool(wmask.all())
    assert torch.equal(a.clients.params[..., ~wmask], b.clients.params[..., ~wmask])   # BatchNorm statistics and counters
    assert not torch.allclose(a.clients.params[..., wmask], b.clients.params[..., wmask])
    one_a, one_b = _resnet_round(5.0, 1), _resnet_round(0.0, 1)
    assert torch.equal(one_a.bank.theta, one_b.bank.theta)


def _trainer(mu, optimizer, epochs):
    from feddrift_b200.drift.fedavg_ens import FedAvgEnsTrainer
    g = torch.Generator().manual_seed(7)
    models = [mutils.create_model("fnn", 2, 3) for _ in range(2)]
    batches = [[(torch.randn(16, 3, generator=g), torch.randint(0, 2, (16,), generator=g))] for _ in range(2)]
    args = _sea(fedprox_mu=mu, client_optimizer=optimizer, epochs=epochs, lr=0.05, wd=1e-3)
    tr = FedAvgEnsTrainer(0, [{0: b} for b in batches], [{0: 16} for _ in batches], None, None, "cpu", models, args)
    return tr, models, batches


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_facade_trainer_equals_a_hand_written_proximal_loop(optimizer):
    tr, models, batches = _trainer(MU, optimizer, 3)
    start = [copy.deepcopy(m) for m in models]
    res = tr.train()
    for i, m0 in enumerate(start):
        anchor = [p.detach().clone() for p in m0.parameters()]
        opt = torch.optim.SGD(m0.parameters(), lr=0.05) if optimizer == "sgd" else \
            torch.optim.Adam(m0.parameters(), lr=0.05, weight_decay=1e-3, amsgrad=True)
        x, y = batches[i][0]
        for _ in range(3):
            opt.zero_grad()
            F.cross_entropy(m0(x), y).backward()
            for p, a in zip(m0.parameters(), anchor):
                p.grad.add_(p.detach() - a, alpha=MU)
            opt.step()
        for k, v in m0.state_dict().items():
            assert torch.equal(res[i][0][k], v), (i, k)
    one, _, _ = _trainer(MU, optimizer, 1)
    zero, _, _ = _trainer(0.0, optimizer, 1)
    ra, rb = one.train(), zero.train()
    for i in ra:
        for k in ra[i][0]:
            assert torch.equal(ra[i][0][k], rb[i][0][k])


def test_checkpoint_resume_with_fedprox(tmp_path):
    kw = dict(dataset="sine", concept_drift_algo_arg="H_A_C_1_0_0", comm_round=6, lr=0.05, total_train_iteration=4, sample_num=60,
              epochs=3, fedprox_mu=MU)
    full = DriftSim(make_args(**kw), device="cpu", sink=MetricsSink())
    full.run()
    part = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    part.run(0, 2)
    resumed = DriftSim(make_args(checkpoint_dir=str(tmp_path), **kw), device="cpu", sink=MetricsSink())
    nxt = checkpoint.resume(resumed, checkpoint.latest(str(tmp_path)))
    assert nxt == 2
    resumed.run(nxt)
    assert torch.allclose(resumed.bank.theta, full.bank.theta, atol=1e-6)


@pytest.mark.parametrize("mu", [-0.1, float("nan"), float("inf")])
def test_rejections(mu):
    with pytest.raises(ValueError):
        DriftSim(_sea(fedprox_mu=mu), device="cpu", sink=MetricsSink())
    with pytest.raises(ValueError):
        _trainer(mu, "adam", 1)
    with pytest.raises(ValueError):
        ref.fed_round_small(with_prox(make_state(C=6, S=20), mu), 1)


def test_cli_flag_and_config():
    from feddrift_b200.experiments.configs import CONFIGS
    from feddrift_b200.experiments.fedavg_cont_ens import add_args
    p = add_args(argparse.ArgumentParser())
    assert p.parse_args([]).fedprox_mu == 0.0
    assert p.parse_args(["--fedprox_mu", "0.01"]).fedprox_mu == 0.01
    assert CONFIGS["cfg2x_sea_fnn_100clients_fedprox_feddrift"]["fedprox_mu"] == 0.1
    assert np.isclose(make_args().fedprox_mu, 0.0)
