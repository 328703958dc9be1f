"""Robust aggregation on the GPU: the fused round kernel's publish-step defense vs the CPU oracle, launch modes and CUDA-graph
replay, the slot-anchored K10 kernel vs its reference, and the generic executor's routes (per-pair graphs, stacked ResNet-18,
batched LSTM) against the reference defense applied to their raw upload arena."""
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

DEFENSES = ["norm_diff_clipping", "weak_dp"]


def with_defense(st, defense, bound=0.1, stddev=0.01):
    return dict(st, defense=defense, norm_bound=bound, stddev=stddev)


def _compare(st_gpu, st_cpu, atol=2e-5):
    assert torch.allclose(st_gpu["theta"].cpu(), st_cpu["theta"], rtol=2e-4, atol=atol), \
        (st_gpu["theta"].cpu() - st_cpu["theta"]).abs().max()
    assert torch.equal(st_gpu["opt_step"].cpu(), st_cpu["opt_step"])


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("defense", DEFENSES)
@pytest.mark.parametrize("cfg", CFGS)
def test_fused_round_with_defense_matches_reference(cfg, defense, table):
    st_cpu = with_defense(make_state(**cfg), defense)
    C = st_cpu["X"].shape[1]
    if table:
        st_cpu["participation"] = _table(3, C, max(1, C // 3))
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu)


@pytest.mark.parametrize("defense", DEFENSES)
def test_fused_round_with_defense_ifca_recluster(defense):
    st_cpu = with_defense(make_state(M=3), defense)
    st_cpu["recluster_hard"] = True
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 2)
    ops.fed_round_small(st_gpu, 2)
    torch.cuda.synchronize()
    assert torch.equal(st_gpu["W"][st_gpu["t_cur"]].cpu(), st_cpu["W"][st_cpu["t_cur"]])
    _compare(st_gpu, st_cpu)


def test_fused_round_with_defense_and_server_adam():
    st_cpu = with_server_opt(with_defense(make_state(), "weak_dp"), "adam")
    st_cpu["participation"] = _table(3, 10, 4)
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu, atol=1e-4)   # Adam scales last-bit differences of the average by up to lr/τ
    assert torch.equal(st_gpu["server_step"].cpu(), st_cpu["server_step"])


def test_unreached_bound_is_bit_identical_to_none():
    st = make_state(C=12)
    st["participation"] = _table(3, 12, 5)
    a = to_cuda(with_defense(copy.deepcopy(st), "norm_diff_clipping", bound=1e30))
    b = to_cuda(copy.deepcopy(st))
    ops.fed_round_small(a, 3)
    ops.fed_round_small(b, 3)
    torch.cuda.synchronize()
    assert torch.equal(a["theta"], b["theta"]) and torch.equal(a["opt_m"], b["opt_m"])


@pytest.mark.parametrize("defense", DEFENSES)
def test_three_rounds_in_one_launch_equal_three_launches(defense):
    st = with_defense(make_state(C=12), defense)
    st["participation"] = _table(3, 12, 4)
    st["client_out"] = torch.zeros(12, *st["theta"].shape)
    one, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_step"):
        assert torch.equal(one[k], three[k]), k
    last = st["participation"][2].bool().cuda()   # every launch exports its last round: compare round 3's participants
    assert torch.equal(one["client_out"][last], three["client_out"][last])


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, defense_type="weak_dp", norm_bound=0.05, stddev=0.01)
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
    plain = _sim(client_num_per_round=3, defense_type="none")
    for t in range(2):
        plain.run_time_step(t, rounds=4)
    assert not torch.allclose(plain.bank.theta, a.bank.theta)


@pytest.mark.parametrize("stddev", [0.0, 0.05])
def test_robust_clip_slots_matches_reference(stddev):
    g = torch.Generator().manual_seed(5)
    C, M, P, stride = 7, 3, 1000, 1024
    bank = torch.randn(M, stride, generator=g)
    theta = bank[:, :P]   # a padded bank: row stride 1024
    up = theta[None] + torch.randn(C, M, P, generator=g) * torch.rand(C, M, 1, generator=g) * 2.0
    n = torch.rand(C, M, generator=g)
    n[n < 0.3] = 0
    mask = torch.rand(P, generator=g) > 0.1
    cpu = up.clone()
    nrm_c = ref.robust_clip_slots_(cpu, theta, n, 20.0, mask, stddev, 77)
    gpu = up.cuda()
    nrm_g = ops.robust_clip_slots_(gpu, bank.cuda()[:, :P], n.cuda(), 20.0, mask.cuda(), stddev, 77)
    torch.cuda.synchronize()
    assert bool((nrm_c > 20.0).any()) and bool(((nrm_c < 20.0) & (n > 0)).any())
    assert torch.allclose(nrm_g.cpu(), nrm_c, rtol=1e-5)
    assert torch.allclose(gpu.cpu(), cpu, rtol=1e-5, atol=1e-5), (gpu.cpu() - cpu).abs().max()
    assert torch.equal(gpu.cpu()[n == 0], up[n == 0])             # weight 0: untouched
    assert torch.equal(gpu.cpu()[..., ~mask], up[..., ~mask])     # masked entries pass through
    if stddev == 0.0:
        keep = (nrm_c < 20.0) & (n > 0)                           # bound not reached, no noise: bit-identical
        assert torch.equal(gpu.cpu()[keep], up[keep])


def _generic_defended(kw, env=None):
    """One round of time step 0 on the generic executor with a defense: the arena the round aggregated must be the reference
    defense of the raw arena training left, and θ its weighted mean."""
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        d = dict(defense_type="weak_dp", norm_bound=0.01, stddev=0.01)
        d.update(kw)
        sim = DriftSim(make_args(**d), device="cuda", sink=MetricsSink())
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        raw = []
        real = sim.defense.defend_slots_

        def spy(up, *a):
            raw.append((up.clone(), a[1].clone()))
            return real(up, *a)
        sim.defense.defend_slots_ = spy
        theta0 = sim.bank.theta.clone()
        sim.run_rounds(1)
        torch.cuda.synchronize()
        up, n = raw[0]
        want_up = up.cpu()
        norms = ref.robust_clip_slots_(want_up, theta0.cpu(), n.cpu(), 0.01, sim.defense_mask, 0.01, ref.defense_seed(13, 0))
        assert bool((norms > 0.01).any())
        sel = n.cpu() > 0
        assert torch.allclose(sim.clients.params.cpu()[sel], want_up[sel], rtol=1e-5, atol=1e-6)
        want = theta0.cpu().clone()
        ref.cluster_aggregate_(want, want_up, n.cpu())
        assert torch.allclose(sim.bank.theta.cpu(), want, rtol=1e-4, atol=1e-5), (sim.bank.theta.cpu() - want).abs().max()
        return sim
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_generic_per_pair_graphs_defend_uploads():
    sim = _generic_defended(dict(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                                 concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                                 total_train_iteration=2, epochs=2))
    assert any(g.indexed and g.launches > 0 for g in sim.__dict__.get("_step_graphs", {}).values()), "per-pair graphs not used"


def test_generic_stacked_resnet_defends_uploads_and_keeps_bn_buffers(monkeypatch):
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    sim = _generic_defended(dict(model="resnet18", dataset="cifar10", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1",
                                 concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=2,
                                 total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05), {"FDB_STACKED": "force"})
    assert calls
    assert sim.defense_mask is not None and not bool(sim.defense_mask.all())


def test_generic_lstm_defends_uploads():
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    _generic_defended(dict(model="rnn", dataset="shakespeare", client_num_in_total=6, concept_num=2, concept_drift_algo="win-1",
                           concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16, comm_round=2,
                           total_train_iteration=2, epochs=2, lr=0.05, client_optimizer="sgd", report_client=0))
    assert fused.CALLS["bwd"] > n0, "batched LSTM executor did not run"


def test_binding_rejects_bad_defense_scalars():
    st = to_cuda(make_state())
    for bound, std in ((float("nan"), 0.0), (-1.0, 0.0), (1.0, -0.5), (1.0, float("inf"))):
        with pytest.raises(ValueError):
            ops.fed_round_small(with_defense(copy.deepcopy(st), "weak_dp", bound, std), 1)
    rows = torch.zeros(2, 2, 8, device="cuda")
    with pytest.raises(RuntimeError):
        ops._ext.load().robust_clip_slots(rows, torch.zeros(3, 8, device="cuda"), None, 1.0, None, 0.0, 0)   # M mismatch
    with pytest.raises(RuntimeError):
        ops._ext.load().robust_clip_slots(rows, torch.zeros(2, 8, device="cuda"), None, 0.0, None, 0.0, 0)   # bound 0


WORKER = r'''
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, os.environ["FDB_ROOT"])
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.parallel.symm import attach_multi_gpu, check_error
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
kw = dict(comm_round=6, total_train_iteration=3, client_num_in_total=10, defense_type="weak_dp", norm_bound=0.05, stddev=0.01)
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
def test_two_gpu_fused_with_defense_matches_single_gpu(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, FDB_ROOT=root, PYTHONFAULTHANDLER="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
