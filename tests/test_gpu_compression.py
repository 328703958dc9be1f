"""QSGD upload compression on the GPU: K17 (``qsgd_slots``) bit for bit against the CPU oracle, the fused round kernel's
publish-step quantizer (exactly against the oracle quantizer applied to its own raw uploads, and against the round oracle over
the fused-round configs, launch modes and CUDA-graph replay), and the generic executor's routes (per-pair graphs, stacked
ResNet-18, batched LSTM)."""
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
from test_robust_defense import _weights
from test_server_opt import with_server_opt

pytestmark = pytest.mark.gpu


def with_q(st, s=65535, b=16):
    return dict(st, compression="qsgd", quantize_level=s, quantize_bucket=b)


def _k17_case(C, M, P, stride, s, b, masked=False, n_zero=True, seed=3):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, stride, generator=g)
    theta = bank[:, :P]
    up = theta[None] + torch.randn(C, M, P, generator=g) * torch.rand(C, M, 1, generator=g)
    up[0, 0, : min(P, 2 * b)] = theta[0, : min(P, 2 * b)]   # zero-update buckets stay unchanged
    n = torch.rand(C, M, generator=g) + 0.1
    if n_zero:
        n[n < 0.4] = 0
    mask = (torch.rand(P, generator=g) > 0.1) if masked else None
    cpu = up.clone()
    ref.qsgd_slots_(cpu, theta, n, s, b, mask, 0xC0FFEE)
    gpu = up.cuda()
    ops.qsgd_slots_(gpu, bank.cuda()[:, :P], n.cuda(), s, b, None if mask is None else mask.cuda(), 0xC0FFEE)
    torch.cuda.synchronize()
    return up, cpu, gpu.cpu(), n, mask


@pytest.mark.parametrize("C,M,P,stride,s,b,masked", [
    (5, 3, 1001, 1001, 4, 64, False),     # odd P, unaligned rows: scalar path
    (5, 3, 1003, 1024, 16, 100, True),    # P not a multiple of b, padded bank, mask
    (4, 2, 1024, 1032, 2, 1, False),      # b = 1, aligned: 128-bit path
    (4, 2, 999, 999, 3, 999, True),       # b = P
    (4, 2, 1000, 1024, 5, 5000, False),   # b > P
    (3, 2, 4096, 4096, 1, 512, True),     # s = 1: ternary
    (3, 2, 4099, 4100, 65535, 37, False), # s = 65535
])
def test_row_qsgd_matches_reference_bit_for_bit(C, M, P, stride, s, b, masked):
    up, cpu, gpu, n, mask = _k17_case(C, M, P, stride, s, b, masked)
    assert torch.equal(gpu, cpu), (gpu != cpu).sum()
    assert torch.equal(gpu[n == 0], up[n == 0])
    if mask is not None:
        assert torch.equal(gpu[..., ~mask], up[..., ~mask])
    if b > 1:   # b = 1: σ = |d| and q = s, so every entry is its own level (θ + d)
        assert not torch.equal(gpu[n > 0], up[n > 0])


def test_row_qsgd_large_row_one_bucket_spans_many_ctas():
    P = (1 << 20) + 12
    up, cpu, gpu, n, _ = _k17_case(2, 2, P, P + 4, 8, 1 << 20, n_zero=False)
    assert torch.equal(gpu, cpu), (gpu != cpu).sum()


def test_row_qsgd_two_launches_are_bit_identical():
    g = torch.Generator().manual_seed(9)
    theta = torch.randn(4, 50000, generator=g).cuda()
    up = theta[None] + torch.randn(8, 4, 50000, generator=g).cuda()
    a, b = up.clone(), up.clone()
    ops.qsgd_slots_(a, theta, None, 4, 512, None, 5)
    ops.qsgd_slots_(b, theta, None, 4, 512, None, 5)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and not torch.equal(a, up)


@pytest.mark.parametrize("s,b", [(2, 16), (4, 7)])
def test_fused_round_quantizes_its_own_uploads_exactly(s, b):
    st = make_state(C=12)
    C, M, P = st["X"].shape[1], *st["theta"].shape
    theta0 = st["theta"].clone()
    st["client_out"] = torch.zeros(C, M, P)
    plain, q = to_cuda(copy.deepcopy(st)), to_cuda(with_q(copy.deepcopy(st), s, b))
    ops.fed_round_small(plain, 1)
    ops.fed_round_small(q, 1)
    torch.cuda.synchronize()
    n = _weights(st)
    want = plain["client_out"].cpu()
    assert bool((want[n > 0] != 0).any())
    ref.qsgd_slots_(want, theta0, n, s, b, None, ref.compress_seed(st["seed"], 0))
    assert torch.equal(q["client_out"].cpu(), want)   # the training paths are the same code: identical raw models
    agg = theta0.clone()
    ref.cluster_aggregate_(agg, want, n)
    assert torch.allclose(q["theta"].cpu(), agg, rtol=1e-5, atol=1e-6)
    assert torch.equal(q["opt_m"], plain["opt_m"])


def _compare(st_gpu, st_cpu, atol=2e-5):
    assert torch.allclose(st_gpu["theta"].cpu(), st_cpu["theta"], rtol=2e-4, atol=atol), \
        (st_gpu["theta"].cpu() - st_cpu["theta"]).abs().max()
    assert torch.equal(st_gpu["opt_step"].cpu(), st_cpu["opt_step"])


# Against the round oracle, local training differs from the CPU in the last bits, and a quantizer turns a last-bit change of
# an input into a one-level change of its output whenever the draw u falls between the two fractions.  These comparisons
# therefore use s = 65535, where one level is σ/65535 and stays inside the existing tolerance; the low-level cases are
# covered exactly by the test above, which quantizes the kernel's own raw uploads.
@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("cfg", CFGS)
def test_fused_round_with_qsgd_matches_reference(cfg, table):
    st_cpu = with_q(make_state(**cfg))
    C = st_cpu["X"].shape[1]
    if table:
        st_cpu["participation"] = _table(3, C, max(1, C // 3))
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu)


def test_fused_round_with_qsgd_ifca_recluster():
    st_cpu = with_q(make_state(M=3))
    st_cpu["recluster_hard"] = True
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 2)
    ops.fed_round_small(st_gpu, 2)
    torch.cuda.synchronize()
    assert torch.equal(st_gpu["W"][st_gpu["t_cur"]].cpu(), st_cpu["W"][st_cpu["t_cur"]])
    _compare(st_gpu, st_cpu)


def test_fused_round_with_qsgd_and_weak_dp():
    st_cpu = dict(with_q(make_state()), defense="weak_dp", norm_bound=0.1, stddev=0.01)
    st_cpu["participation"] = _table(3, 10, 4)
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu)


def test_fused_round_with_qsgd_and_server_adam():
    st_cpu = with_server_opt(with_q(make_state()), "adam")
    st_cpu["participation"] = _table(3, 10, 4)
    st_gpu = to_cuda(copy.deepcopy(st_cpu))
    ref.fed_round_small(st_cpu, 3)
    ops.fed_round_small(st_gpu, 3)
    torch.cuda.synchronize()
    _compare(st_gpu, st_cpu, atol=1e-4)   # Adam scales last-bit differences of the average by up to lr/τ
    assert torch.equal(st_gpu["server_step"].cpu(), st_cpu["server_step"])


def test_three_rounds_in_one_launch_equal_three_launches():
    st = with_q(make_state(C=12), 2, 16)
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
    d = dict(comm_round=6, total_train_iteration=4, compression="qsgd", quantize_level=2, quantize_bucket=16)
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
    plain = _sim(client_num_per_round=3, compression="none")
    for t in range(2):
        plain.run_time_step(t, rounds=4)
    assert not torch.allclose(plain.bank.theta, a.bank.theta)


def _generic_quantized(kw, env=None, s=2, b=64):
    """One round of time step 0 on the generic executor with QSGD: the arena the round aggregated must be the reference
    quantizer applied to the raw arena training left (bit for bit: K17 is exact), and θ its weighted mean."""
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        d = dict(compression="qsgd", quantize_level=s, quantize_bucket=b)
        d.update(kw)
        sim = DriftSim(make_args(**d), device="cuda", sink=MetricsSink())
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        raw = []
        real = ops.qsgd_slots_

        def spy(rows, theta, n, *a):
            raw.append((rows.clone(), n.clone()))
            return real(rows, theta, n, *a)
        ops.qsgd_slots_ = spy
        try:
            theta0 = sim.bank.theta.clone()
            sim.run_rounds(1)
            torch.cuda.synchronize()
        finally:
            ops.qsgd_slots_ = real
        up, n = raw[0]
        want_up = up.cpu()
        mask = None if sim.defense_mask is None else sim.defense_mask.cpu()
        ref.qsgd_slots_(want_up, theta0.cpu(), n.cpu(), s, b, mask, ref.compress_seed(13, 0))
        assert torch.equal(sim.clients.params.cpu(), want_up)
        sel = n.cpu() > 0
        assert not torch.equal(want_up[sel], up.cpu()[sel])
        if mask is not None:   # BatchNorm statistics pass through
            assert torch.equal(want_up[..., ~mask], up.cpu()[..., ~mask])
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


def test_generic_per_pair_graphs_quantize_uploads():
    sim = _generic_quantized(dict(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                                  concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                                  total_train_iteration=2, epochs=2))
    assert any(g.indexed and g.launches > 0 for g in sim.__dict__.get("_step_graphs", {}).values()), "per-pair graphs not used"


def test_generic_stacked_resnet_quantizes_uploads_and_keeps_bn_buffers(monkeypatch):
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    sim = _generic_quantized(dict(model="resnet18", dataset="cifar10", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1",
                                  concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=2,
                                  total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05), {"FDB_STACKED": "force"},
                             s=4, b=512)
    assert calls
    assert sim.defense_mask is not None and not bool(sim.defense_mask.all())


def test_generic_lstm_quantizes_uploads():
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    _generic_quantized(dict(model="rnn", dataset="shakespeare", client_num_in_total=6, concept_num=2, concept_drift_algo="win-1",
                            concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16, comm_round=2,
                            total_train_iteration=2, epochs=2, lr=0.05, client_optimizer="sgd", report_client=0))
    assert fused.CALLS["bwd"] > n0, "batched LSTM executor did not run"


def test_binding_rejects_bad_scalars():
    st = to_cuda(make_state())
    for s, b in ((0, 16), (65536, 16), (2.5, 16), (4, 0)):
        with pytest.raises(ValueError):
            ops.fed_round_small(with_q(copy.deepcopy(st), s, b), 1)
    ext = ops._ext.load()
    rows = torch.zeros(2, 2, 8, device="cuda")
    theta = torch.zeros(2, 8, device="cuda")
    for level, bucket, seed in ((0, 4, 0), (65536, 4, 0), (4, 0, 0), (4, 4, -1), (4, 4, 1 << 32)):
        with pytest.raises(RuntimeError):
            ext.qsgd_slots(rows, theta, None, level, bucket, None, seed)
    with pytest.raises(RuntimeError):
        ext.qsgd_slots(rows, torch.zeros(3, 8, device="cuda"), None, 4, 4, None, 0)   # M mismatch
    with pytest.raises(RuntimeError):
        ext.qsgd_slots(rows, theta, torch.ones(3, device="cuda"), 4, 4, None, 0)      # n of the wrong size


WORKER = r'''
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, os.environ["FDB_ROOT"])
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.parallel.symm import attach_multi_gpu, check_error
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
kw = dict(comm_round=6, total_train_iteration=3, client_num_in_total=10, compression="qsgd", quantize_level=65535, quantize_bucket=16)
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
def test_two_gpu_fused_with_qsgd_matches_single_gpu(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, FDB_ROOT=root, PYTHONFAULTHANDLER="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
