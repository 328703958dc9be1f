"""Partial client participation on the GPU: the fused round kernel with a participation table vs the CPU oracle, per-round
prep inside one launch, CUDA-graph replay, the generic executor's routes and the two-rank fused mode."""
import copy
import os
import subprocess
import sys

import pytest
import torch

from feddrift_b200 import ops
from feddrift_b200.ops import reference as ref
from feddrift_b200.sim.sampling import sample_clients
from test_gpu_small_round import make_state, to_cuda

pytestmark = pytest.mark.gpu


def _table(rows, C, K):
    tab = torch.zeros(rows, C, dtype=torch.uint8)
    for r in range(rows):
        tab[r, torch.from_numpy(sample_clients(r, C, K))] = 1
    return tab


@pytest.mark.parametrize("cfg", [
    dict(), dict(optimizer="sgd"), dict(kind="lr", hid=0), dict(din=2, hid=4), dict(B=32), dict(mode="time"),
    dict(mode="index", B=64), dict(C=37, M=4), dict(kind="fnn", din=4, hid=8, dout=3),
])
def test_fused_round_with_table_matches_reference(cfg):
    st_cpu = make_state(**cfg)
    C = st_cpu["X"].shape[1]
    st_cpu["participation"] = _table(3, C, max(1, C // 3))
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    before = copy.deepcopy(st_cpu)
    rounds = 3
    out_ref = ref.fed_round_small(st_cpu, rounds)
    out_gpu = ops.fed_round_small(st_gpu, rounds)
    torch.cuda.synchronize()
    assert torch.allclose(st_gpu["theta"].cpu(), st_cpu["theta"], rtol=2e-4, atol=2e-5), \
        (st_gpu["theta"].cpu() - st_cpu["theta"]).abs().max()
    assert torch.equal(st_gpu["opt_step"].cpu(), st_cpu["opt_step"])
    if st_cpu["optimizer"] == "adam":
        assert torch.allclose(st_gpu["opt_m"].cpu(), st_cpu["opt_m"], rtol=1e-3, atol=1e-6)
    mg, mr = out_gpu["metrics"].cpu(), out_ref["metrics"]
    assert (mg[..., 0] - mr[..., 0]).abs().max() <= 1.0
    assert torch.allclose(mg[..., 1], mr[..., 1], rtol=1e-3, atol=1e-2)
    assert (mg[..., 2] - mr[..., 2]).abs().max() <= 1.0
    assert torch.allclose(out_gpu["counts"].cpu(), out_ref["counts"])
    # clients outside every row keep their optimizer state bit for bit
    never = st_cpu["participation"].sum(0) == 0
    for k in ("opt_m", "opt_v", "opt_vmax", "opt_step"):
        assert torch.equal(st_gpu[k].cpu()[never], before[k][never]), k


def test_fused_round_with_table_ifca_recluster():
    st_cpu = make_state(M=3)
    st_cpu["recluster_hard"] = True
    st_cpu["participation"] = _table(2, 10, 3)
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 2)
    ops.fed_round_small(st_gpu, 2)
    torch.cuda.synchronize()
    Wg = st_gpu["W"][st_gpu["t_cur"]].cpu()
    assert torch.all(Wg.sum(0) == 1)
    agree = (Wg.argmax(0) == st_cpu["W"][st_cpu["t_cur"]].argmax(0)).float().mean()
    assert agree >= 0.8
    assert torch.equal(st_gpu["opt_step"].cpu(), st_cpu["opt_step"])


def test_all_ones_table_equals_no_table_on_gpu():
    st = to_cuda(make_state())
    a, b = copy.deepcopy(st), copy.deepcopy(st)
    b["participation"] = torch.ones(2, 10, dtype=torch.uint8, device="cuda")
    oa, ob = ops.fed_round_small(a, 3), ops.fed_round_small(b, 3)
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_v", "opt_vmax", "opt_step"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(oa["metrics"], ob["metrics"])


def test_three_rounds_in_one_launch_equal_three_launches():
    st = make_state(C=12)
    st["participation"] = _table(3, 12, 4)
    one, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    m_one = ops.fed_round_small(one, 3)["metrics"].clone()
    m_three = torch.cat([ops.fed_round_small(three, 1)["metrics"].clone() for _ in range(3)])
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_v", "opt_vmax", "opt_step"):
        assert torch.equal(one[k], three[k]), k
    assert torch.equal(m_one, m_three)
    # and the table mattered: a launch that (wrongly) reused row 0 for every round gives other models
    row0 = to_cuda(copy.deepcopy(st))
    row0["participation"] = row0["participation"][:1].contiguous()
    ops.fed_round_small(row0, 3)
    assert not torch.equal(row0["theta"], one["theta"])


def test_round_graph_follows_device_round_counter_under_sampling():
    from feddrift_b200.sim import DriftSim, make_args

    def make():
        sim = DriftSim(make_args(comm_round=6, total_train_iteration=4, client_num_per_round=3), device="cuda")
        for t in range(2):
            sim.run_time_step(t, rounds=4)
        sim.begin_time_step(2)
        sim.args.rounds_per_launch = 1
        return sim

    a, b = make(), make()
    assert a.participation is not None
    ha, hb = a.make_host_round_inputs(), b.make_host_round_inputs()
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert torch.allclose(a.bank.theta, b.bank.theta, atol=1e-6)
    assert torch.equal(a.clients.step, b.clients.step)
    seen = torch.from_numpy(a.participation[:4].any(0))
    trained = (a.clients.step > 0).any(1).cpu()
    assert trained.any() and not (trained & ~seen).any()


def _generic_rounds(kw, rounds, env=None):
    """Run ``rounds`` single-round blocks of time step 0 and check every round against the participation table."""
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        for r in range(rounds):
            theta0 = sim.bank.theta.clone()
            sim.run_rounds(1)
            torch.cuda.synchronize()
            row = torch.from_numpy(sim.participants(r))
            n = sim.clients.n.cpu()
            trained = (n > 0).any(1)
            assert trained.any() and not (trained & ~row).any(), (r, trained, row)
            for m in range(sim.M):
                if not (n[:, m] > 0).any():
                    assert torch.equal(sim.bank.theta[m], theta0[m]), (r, m)
                else:
                    assert not torch.equal(sim.bank.theta[m], theta0[m]), (r, m)
        sim.end_time_step()
        return sim
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_generic_per_pair_graphs_follow_table():
    sim = _generic_rounds(dict(model="fnn", dataset="MNIST", client_num_in_total=6, client_num_per_round=2, concept_num=2,
                               concept_drift_algo="softcluster", concept_drift_algo_arg="H_A_C_1_10_0", change_points="A",
                               sample_num=16, batch_size=8, comm_round=3, total_train_iteration=2, epochs=2), 3)
    assert any(g.indexed and g.launches > 0 for g in sim.__dict__.get("_step_graphs", {}).values()), "per-pair graphs not used"


def test_generic_stacked_resnet_follows_table(monkeypatch):
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    _generic_rounds(dict(model="resnet18", dataset="cifar10", client_num_in_total=4, client_num_per_round=2, concept_num=2,
                         concept_drift_algo="win-1", concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8,
                         comm_round=2, total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05), 2,
                    {"FDB_STACKED": "force"})
    assert calls and all(n <= 2 for n in calls), calls


def test_generic_lstm_follows_table():
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    _generic_rounds(dict(model="rnn", dataset="shakespeare", client_num_in_total=6, client_num_per_round=2, concept_num=2,
                         concept_drift_algo="win-1", concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16,
                         comm_round=2, total_train_iteration=2, epochs=2, lr=0.05, client_optimizer="sgd", report_client=0), 2)
    assert fused.CALLS["bwd"] > n0, "batched LSTM executor did not run"


WORKER = r'''
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, os.environ["FDB_ROOT"])
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.parallel.symm import attach_multi_gpu, check_error
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
kw = dict(comm_round=6, total_train_iteration=3, client_num_in_total=10, client_num_per_round=3)
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
def test_two_gpu_fused_with_table_matches_single_gpu(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, FDB_ROOT=root, PYTHONFAULTHANDLER="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29537", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
