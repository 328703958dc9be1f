"""FedProx local training on the GPU: the fused round kernel's proximal term vs the CPU oracle, launch modes and CUDA-graph
replay, the anchored row optimizers vs their references, and the generic executor's routes (per-pair graphs, eager, stacked
ResNet-18, batched LSTM with Adam and SGD) against the eager per-pair path."""
import copy
import os
import subprocess
import sys

import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from test_gpu_server_opt import CFGS, _table
from test_gpu_small_round import make_state, to_cuda
from test_server_opt import with_server_opt

pytestmark = pytest.mark.gpu

MU = 0.1


def with_prox(st, mu=MU):
    return dict(st, fedprox_mu=mu)


def _compare(st_gpu, st_cpu, atol=2e-5):
    assert torch.allclose(st_gpu["theta"].cpu(), st_cpu["theta"], rtol=2e-4, atol=atol), \
        (st_gpu["theta"].cpu() - st_cpu["theta"]).abs().max()
    assert torch.equal(st_gpu["opt_step"].cpu(), st_cpu["opt_step"])


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("cfg", CFGS)
def test_fused_round_with_fedprox_matches_reference(cfg, table):
    st_cpu = with_prox(make_state(**cfg))
    C = st_cpu["X"].shape[1]
    if table:
        st_cpu["participation"] = _table(3, C, max(1, C // 3))
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu)


def test_fused_round_with_fedprox_ifca_recluster():
    st_cpu = with_prox(make_state(M=3))
    st_cpu["recluster_hard"] = True
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 2)
    ops.fed_round_small(st_gpu, 2)
    torch.cuda.synchronize()
    assert torch.equal(st_gpu["W"][st_gpu["t_cur"]].cpu(), st_cpu["W"][st_cpu["t_cur"]])
    _compare(st_gpu, st_cpu)


def test_fused_round_with_fedprox_server_adam_and_weak_dp():
    st_cpu = with_prox(with_server_opt(dict(make_state(), defense="weak_dp", norm_bound=0.1, stddev=0.01), "adam"))
    st_cpu["participation"] = _table(3, 10, 4)
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu, atol=1e-4)   # Adam scales last-bit differences of the average by up to lr/τ
    assert torch.equal(st_gpu["server_step"].cpu(), st_cpu["server_step"])


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_fused_mu_zero_and_one_step_are_bit_identical(optimizer):
    st = make_state(C=12, optimizer=optimizer)
    st["participation"] = _table(3, 12, 5)
    a, b = to_cuda(with_prox(copy.deepcopy(st), 0.0)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(a, 3)
    ops.fed_round_small(b, 3)
    one = make_state(C=12, optimizer=optimizer, epochs=1)
    c, d = to_cuda(with_prox(copy.deepcopy(one))), to_cuda(copy.deepcopy(one))
    ops.fed_round_small(c, 3)
    ops.fed_round_small(d, 3)
    e = to_cuda(with_prox(copy.deepcopy(st)))
    ops.fed_round_small(e, 3)
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_step"):
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(c[k], d[k]), k
    assert not torch.equal(e["theta"], b["theta"])


def test_three_rounds_in_one_launch_equal_three_launches():
    st = with_prox(make_state(C=12))
    st["participation"] = _table(3, 12, 4)
    st["client_out"] = torch.zeros(12, *st["theta"].shape)
    one, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_step"):
        assert torch.equal(one[k], three[k]), k
    last = st["participation"][2].bool().cuda()
    assert torch.equal(one["client_out"][last], three["client_out"][last])


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, fedprox_mu=MU)
    d.update(kw)
    return DriftSim(make_args(**d), device="cuda", sink=MetricsSink())


def test_round_graph_replay_matches_non_graph_path():
    def make():
        sim = _sim(client_num_per_round=3)
        for t in range(2):
            sim.run_time_step(t, rounds=4)
        sim.begin_time_step(2)
        sim.args.rounds_per_launch = 1
        return sim

    a, b = make(), make()
    ha, hb = a.make_host_round_inputs(), b.make_host_round_inputs()
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert torch.equal(a.bank.theta, b.bank.theta)
    plain = _sim(client_num_per_round=3, fedprox_mu=0.0)
    for t in range(2):
        plain.run_time_step(t, rounds=4)
    assert not torch.allclose(plain.bank.theta, a.bank.theta)


@pytest.mark.parametrize("P", [1000, 1001])
@pytest.mark.parametrize("opt", ["adam", "sgd"])
def test_row_optimizers_with_prox_match_reference(opt, P):
    g = torch.Generator().manual_seed(11)
    R, A, stride = 6, 3, 1032
    bank = torch.randn(A, stride, generator=g)
    anchor = bank[:, :P]   # a padded bank: row stride 1032
    rows = torch.tensor([2, 0, 1, 2, 0, 1], dtype=torch.int32)
    mask = (torch.rand(P, generator=g) > 0.2).to(torch.uint8)
    row_mask = torch.tensor([1, 1, 0, 1, 0, 1], dtype=torch.uint8)
    p0 = anchor[rows.long()] + 0.5 * torch.randn(R, P, generator=g)
    grad = torch.randn(R, P, generator=g)
    state = [torch.rand(R, P, generator=g) * 0.1 for _ in range(3)]
    state[2] = torch.maximum(state[2], state[1])
    steps = torch.tensor([0, 3, 1, 7, 2, 5], dtype=torch.int32)

    def run(dev, prox):
        p, st_, s = p0.clone().to(dev), [x.clone().to(dev) for x in state], steps.clone().to(dev)
        px = None if prox is None else (MU, bank.to(dev)[:, :P], rows.to(dev), mask.to(dev))
        if opt == "adam":
            ops.adam_amsgrad_rows_(p, grad.clone().to(dev), *st_, s, 0.01, 1e-3, row_mask=row_mask.to(dev), prox=px)
        else:
            ops.sgd_rows_(p, grad.clone().to(dev), 0.05, row_mask=row_mask.to(dev), prox=px)
        return p.cpu(), [x.cpu() for x in st_], s.cpu()

    pc, sc, kc = run("cpu", True)
    pg, sg, kg = run("cuda", True)
    torch.cuda.synchronize()
    assert torch.allclose(pg, pc, rtol=1e-5, atol=1e-6), (pg - pc).abs().max()
    for a, b in zip(sg, sc):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7)
    assert torch.equal(kg, kc)
    pn, sn, kn = run("cuda", None)   # masked rows and masked entries: bit-identical to a call without prox
    off = ~row_mask.bool()
    assert torch.equal(pg[off], p0[off]) and torch.equal(pn[off], p0[off])
    on = row_mask.bool()
    emask = ~mask.bool()
    assert torch.equal(pg[on][:, emask], pn[on][:, emask])
    for a, b in zip(sg, sn):
        assert torch.equal(a[on][:, emask], b[on][:, emask])
    assert not torch.equal(pg[on][:, mask.bool()], pn[on][:, mask.bool()])


def _generic_theta(kw, env=None):
    """θ after one round of time step 0 on the generic executor, under the environment ``env``."""
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        sim.run_rounds(1)
        torch.cuda.synchronize()
        return sim
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _check_route(kw, env, eager_env=None, tol=2e-2, entries=None):
    """With E = 2 the route matches the eager per-pair path (on ``entries``, default all) and differs from μ = 0; with E = 1 it is
    bit-identical to μ = 0 (on a route that is itself bit-reproducible)."""
    eager_env = dict({"FDB_NO_GRAPHS": "1"}, **(eager_env or {}))
    k2 = dict(kw, epochs=2, fedprox_mu=1.0)
    sim = _generic_theta(k2, env)
    eager = _generic_theta(k2, eager_env)
    zero = _generic_theta(dict(k2, fedprox_mu=0.0), env)
    th, te, t0 = sim.bank.theta, eager.bank.theta, zero.bank.theta
    if entries is not None:
        th, te, t0 = th[:, entries], te[:, entries], t0[:, entries]
    scale = te.abs().max().item()
    assert (th - te).abs().max().item() < tol * scale, (th - te).abs().max().item()
    assert not torch.allclose(th, t0)
    one = _generic_theta(dict(kw, epochs=1, fedprox_mu=1.0), env)
    one0 = _generic_theta(dict(kw, epochs=1, fedprox_mu=0.0), env)
    if torch.equal(one.bank.theta, one0.bank.theta):
        return sim, zero
    # a route whose own runs differ (atomic gradient accumulation): the μ = 0 run repeated bounds what E = 1 may differ by
    again = _generic_theta(dict(kw, epochs=1, fedprox_mu=0.0), env)
    noise = (again.bank.theta - one0.bank.theta).abs().max().item()
    assert noise > 0, "E = 1 with mu > 0 differs from mu = 0 on a bit-reproducible route"
    assert (one.bank.theta - one0.bank.theta).abs().max().item() <= 4 * noise
    return sim, zero


FNN = dict(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
           concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3, total_train_iteration=2)


def test_generic_per_pair_graphs_with_fedprox():
    sim, _ = _check_route(FNN, None, tol=1e-4)
    assert any(g.indexed and g.launches > 0 for g in sim.__dict__.get("_step_graphs", {}).values()), "per-pair graphs not used"


def test_generic_eager_with_fedprox():
    _check_route(dict(FNN, client_optimizer="sgd", lr=0.05), {"FDB_NO_GRAPHS": "1"}, tol=1e-6)


def test_generic_stacked_resnet_with_fedprox_keeps_bn_buffers(monkeypatch):
    from feddrift_b200.models import utils as mutils
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    kw = dict(model="resnet18", dataset="cifar10", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1",
              concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=2, total_train_iteration=2,
              client_optimizer="sgd", lr=0.05)
    from feddrift_b200.models.utils import create_model
    from feddrift_b200.parallel.arena import ModelBank
    bank = ModelBank(create_model("resnet18", 10, 3, small_input=True), 1, "cpu")
    wmask = mutils.weight_param_mask(bank.spec)[: bank.P].cuda()
    # the BatchNorm batch counters are kept per route (stacked: per pass), so the routes are compared on the weights
    sim, zero = _check_route(kw, {"FDB_STACKED": "force"}, {"FDB_STACKED": "0"}, entries=wmask)
    assert calls and sim.bank.P == bank.P
    assert not bool(wmask.all())
    # BatchNorm statistics get no proximal term (exact on the CPU, test_fedprox.py); this route accumulates its conv weight
    # gradients atomically, so two of its runs agree to the route tolerance only
    bn, bn0 = sim.clients.params[..., ~wmask], zero.clients.params[..., ~wmask]
    assert (bn - bn0).abs().max().item() < 2e-2 * bn0.abs().max().item()


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
def test_generic_lstm_with_fedprox(optimizer):
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    kw = dict(model="rnn", dataset="shakespeare", client_num_in_total=6, concept_num=2, concept_drift_algo="win-1",
              concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16, comm_round=2, total_train_iteration=2,
              lr=0.05 if optimizer == "sgd" else 0.01, client_optimizer=optimizer, report_client=0)
    _check_route(kw, None, {"FDB_LSTM_BATCHED": "0"})
    assert fused.CALLS["bwd"] > n0, "batched LSTM executor did not run"


def test_binding_rejects_bad_mu():
    st = to_cuda(make_state())
    for mu in (-0.1, float("nan"), float("inf")):
        with pytest.raises(RuntimeError):
            ops.fed_round_small(with_prox(copy.deepcopy(st), mu), 1)
    p = torch.zeros(2, 8, device="cuda")
    rows = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        ops._ext.load().sgd_rows(p, p, 0.1, 0.0, None, -1.0, p, rows, None)
    with pytest.raises(RuntimeError):
        ops._ext.load().sgd_rows(p, p, 0.1, 0.0, None, 1.0, p, None, None)   # anchor without anchor_rows


WORKER = r'''
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, os.environ["FDB_ROOT"])
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.parallel.symm import attach_multi_gpu, check_error
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
kw = dict(comm_round=6, total_train_iteration=3, client_num_in_total=10, fedprox_mu=0.1)
sim = DriftSim(make_args(**kw), device=f"cuda:{rank}")
attach_multi_gpu(sim, world, rank)
out = sim.run()
check_error(sim)
ref = DriftSim(make_args(**kw), device=f"cuda:{rank}")
oref = ref.run()
err = (sim.bank.theta - ref.bank.theta).abs().max().item()
gathered = [torch.zeros_like(sim.bank.theta) for _ in range(world)]
dist.all_gather(gathered, sim.bank.theta.contiguous())
same = all(torch.equal(gathered[0], g) for g in gathered)
ok = same and err < 1e-4 and abs(out["history"][-1]["train_acc"] - oref["history"][-1]["train_acc"]) < 0.02
print(json.dumps({"rank": rank, "err": err, "ranks_identical": same, "ok": bool(ok)}))
dist.destroy_process_group()
sys.exit(0 if ok else 3)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_gpu_fused_with_fedprox_matches_single_gpu(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, FDB_ROOT=root, PYTHONFAULTHANDLER="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
