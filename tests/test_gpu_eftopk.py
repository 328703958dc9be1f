"""Top-k sparsification with error feedback on the GPU: K18 (``eftopk_slots``) bit for bit against the CPU oracle, the fused
round kernel's publish-step selection (exactly against the oracle applied to the kernel's own raw uploads, round after round,
over the fused-round configs and with re-clustering, weak DP, a server optimizer and FedProx), launch modes, CUDA-graph
replay, and the generic executor's routes (per-pair graphs, stacked ResNet-18, batched LSTM)."""
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


def with_ef(st, rho=0.3):
    return dict(st, compression="eftopk", topk_ratio=rho)


def _k18_case(C, M, P, stride, k, masked=False, n_zero=True, ties=False, seed=3):
    g = torch.Generator().manual_seed(seed)
    bank = torch.randn(M, stride, generator=g)
    theta = bank[:, :P]
    if ties:   # few distinct magnitudes: the threshold key is shared by many entries spread over the row
        mag = torch.tensor([0.0, 0.25, 0.5, 1.0])[torch.randint(0, 4, (C, M, P), generator=g)]
        up = theta[None] + torch.where(torch.rand(C, M, P, generator=g) < 0.5, -mag, mag)
        res = torch.zeros(C, M, P)
    else:
        up = theta[None] + torch.randn(C, M, P, generator=g) * torch.rand(C, M, 1, generator=g)
        res = 0.1 * torch.randn(C, M, P, generator=g)
        res[torch.rand(C, M, P, generator=g) < 0.3] = 0.0
    n = torch.rand(C, M, generator=g) + 0.1
    if n_zero:
        n[n < 0.4] = 0
    mask = (torch.rand(P, generator=g) > 0.1) if masked else None
    if mask is not None:
        res[..., ~mask] = 0.0
    cpu, cres = up.clone(), res.clone()
    ref.eftopk_slots_(cpu, theta, cres, n, k, mask)
    gpu, gres = up.cuda(), res.cuda()
    ops.eftopk_slots_(gpu, bank.cuda()[:, :P], gres, n.cuda(), k, None if mask is None else mask.cuda())
    torch.cuda.synchronize()
    return up, res, cpu, cres, gpu.cpu(), gres.cpu(), n, mask


@pytest.mark.parametrize("C,M,P,stride,k,masked,ties", [
    (5, 3, 1001, 1001, 10, False, False),    # odd P, unaligned rows: scalar path
    (5, 3, 1003, 1024, 100, True, False),    # padded bank, mask
    (4, 2, 1024, 1032, 1, False, False),     # k = 1, aligned: 128-bit path
    (4, 2, 4096, 4096, 700, False, True),    # forced ties at the threshold
    (4, 2, 4099, 4100, 2000, True, True),    # ties, mask, scalar path
    (3, 2, 999, 999, 999, False, False),     # k = P: every entry kept, no selection
    (3, 2, 1000, 1024, 950, True, False),    # k ≥ trainable count under a mask
    (3, 2, 2048, 2048, 2047, False, False),  # all but one
])
def test_row_eftopk_matches_reference_bit_for_bit(C, M, P, stride, k, masked, ties):
    up, res, cpu, cres, gpu, gres, n, mask = _k18_case(C, M, P, stride, k, masked, ties=ties)
    assert torch.equal(gpu, cpu), (gpu != cpu).sum()
    assert torch.equal(gres, cres), (gres != cres).sum()
    assert torch.equal(gpu[n == 0], up[n == 0]) and torch.equal(gres[n == 0], res[n == 0])
    if mask is not None:
        assert torch.equal(gpu[..., ~mask], up[..., ~mask]) and bool((gres[..., ~mask] == 0).all())


def test_row_eftopk_large_row_spans_many_ctas_and_two_launches_agree():
    P = 11 * (1 << 20) + 3   # a ResNet-18-sized row, odd length
    g = torch.Generator().manual_seed(5)
    theta = torch.randn(1, P + 5, generator=g)
    up = theta[None, :, :P] + 0.01 * torch.randn(2, 1, P, generator=g)
    up[0, 0, 1000:200000] = theta[0, 1000:200000] + 0.0078125   # a block of equal keys around the threshold
    res = torch.zeros(2, 1, P)
    k = 150000
    cpu, cres = up.clone(), res.clone()
    ref.eftopk_slots_(cpu, theta, cres, None, k)
    outs = []
    for _ in range(2):
        gpu, gres = up.cuda(), res.cuda()
        ops.eftopk_slots_(gpu, theta.cuda()[:, :P], gres, None, k)
        torch.cuda.synchronize()
        outs.append((gpu.cpu(), gres.cpu()))
    assert torch.equal(outs[0][0], cpu) and torch.equal(outs[0][1], cres)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_binding_rejects_bad_input():
    ext = ops._ext.load()
    rows = torch.zeros(2, 2, 8, device="cuda")
    theta = torch.zeros(2, 8, device="cuda")
    res = torch.zeros(2, 2, 8, device="cuda")
    with pytest.raises(RuntimeError):
        ext.eftopk_slots(rows, theta, res, None, 0, None)                            # k < 1
    with pytest.raises(RuntimeError):
        ext.eftopk_slots(rows, torch.zeros(3, 8, device="cuda"), res, None, 2, None)  # M mismatch
    with pytest.raises(RuntimeError):
        ext.eftopk_slots(rows, theta, torch.zeros(2, 2, 7, device="cuda"), None, 2, None)   # residual shape
    with pytest.raises(RuntimeError):
        ext.eftopk_slots(rows, theta, res, torch.ones(3, device="cuda"), 2, None)     # n of the wrong size
    st = to_cuda(make_state())
    for rho in (0.0, 1.5, float("nan")):
        with pytest.raises(ValueError):
            ops.fed_round_small(with_ef(copy.deepcopy(st), rho), 1)


def _cpu(st):
    return {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in st.items()}


def _round_against_own_uploads(st, check_theta=None):
    """One fused round of ``st`` (CUDA, eftopk): its uploads and residual must equal the oracle's ``eftopk_slots_`` applied
    to the raw uploads of the same round without compression (local training is the same code in both instantiations) and
    the residual the round started from, bit for bit.  ``check_theta(theta0, uploads, n, st_before)`` checks θ."""
    C, M, P = st["X"].shape[1], *st["theta"].shape
    if st.get("ef_residual") is None:
        st["ef_residual"] = torch.zeros(C, M, P, device="cuda")
    before = _cpu(copy.deepcopy(st))
    plain = copy.deepcopy(st)
    plain.pop("compression")
    plain.pop("ef_residual")
    plain["client_out"] = torch.zeros(C, M, P, device="cuda")
    st["client_out"] = torch.zeros(C, M, P, device="cuda")
    ops.fed_round_small(plain, 1)
    ops.fed_round_small(st, 1)
    torch.cuda.synchronize()
    raw = plain["client_out"].cpu()
    sel = (raw != 0).any(-1)
    assert bool(sel.any())
    want, want_res = raw.clone(), before["ef_residual"].clone()
    ref.eftopk_slots_(want, before["theta"], want_res, sel.float(), ref.topk_k(st["topk_ratio"], P))
    assert torch.equal(st["client_out"].cpu()[sel], want[sel])
    assert torch.equal(st["ef_residual"].cpu(), want_res)
    assert torch.equal(st["opt_m"].cpu(), plain["opt_m"].cpu())
    if check_theta is not None:
        check_theta(before["theta"], want, sel, before)
    return want_res


def _fedavg_theta(rnd_table=None):
    def check(theta0, up, sel, before):
        n = _weights(before) * sel.float()
        want = theta0.clone()
        ref.cluster_aggregate_(want, up, n)
        got = before["_after_theta"]
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (got - want).abs().max()
    return check


def _run_rounds(st, rounds, check=None):
    res = None
    for _ in range(rounds):
        if check is not None:
            holder = {}

            def wrapped(theta0, up, sel, before):
                holder.update(theta0=theta0, up=up, sel=sel, before=before)
            res = _round_against_own_uploads(st, wrapped)
            holder["before"]["_after_theta"] = st["theta"].cpu()
            check(holder["theta0"], holder["up"], holder["sel"], holder["before"])
        else:
            res = _round_against_own_uploads(st)
    assert bool((res != 0).any())
    return res


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("cfg", CFGS)
def test_fused_round_with_eftopk_matches_reference(cfg, table):
    st = with_ef(make_state(**cfg))
    C = st["X"].shape[1]
    if table:
        st["participation"] = _table(3, C, max(1, C // 3))
    _run_rounds(to_cuda(st), 3, _fedavg_theta())


def test_fused_round_with_eftopk_ifca_recluster():
    st = with_ef(make_state(M=3))
    st["recluster_hard"] = True
    _run_rounds(to_cuda(st), 2)


def test_fused_round_with_eftopk_and_weak_dp():
    st = dict(with_ef(make_state()), defense="weak_dp", norm_bound=0.1, stddev=0.01)
    st["participation"] = _table(3, 10, 4)

    def check(theta0, up, sel, before):
        n = _weights(before) * sel.float()
        u = up.clone()
        ref.robust_clip_slots_(u, theta0, n, 0.1, None, 0.01, ref.defense_seed(before["seed"], int(before["round0"])))
        want = theta0.clone()
        ref.cluster_aggregate_(want, u, n)
        assert torch.allclose(before["_after_theta"], want, rtol=1e-5, atol=1e-5)
    _run_rounds(to_cuda(st), 3, check)


def test_fused_round_with_eftopk_server_adam_and_fedprox():
    st = with_server_opt(with_ef(make_state()), "adam")
    st["participation"] = _table(3, 10, 4)
    _run_rounds(to_cuda(st), 3)
    _run_rounds(to_cuda(dict(with_ef(make_state()), fedprox_mu=0.1)), 3)


def test_ratio_one_equals_none_on_the_fused_kernel():
    st = to_cuda(make_state(C=12))
    a, b = with_ef(copy.deepcopy(st), 1.0), copy.deepcopy(st)
    ops.fed_round_small(a, 3)
    ops.fed_round_small(b, 3)
    torch.cuda.synchronize()
    assert torch.equal(a["theta"], b["theta"]) and bool((a["ef_residual"] == 0).all())


def test_three_rounds_in_one_launch_equal_three_launches():
    st = with_ef(make_state(C=12), 0.2)
    st["participation"] = _table(3, 12, 4)
    st["client_out"] = torch.zeros(12, *st["theta"].shape)
    one, three = to_cuda(copy.deepcopy(st)), to_cuda(copy.deepcopy(st))
    ops.fed_round_small(one, 3)
    for _ in range(3):
        ops.fed_round_small(three, 1)
    torch.cuda.synchronize()
    for k in ("theta", "opt_m", "opt_step", "ef_residual"):
        assert torch.equal(one[k], three[k]), k
    last = st["participation"][2].bool().cuda()
    assert torch.equal(one["client_out"][last], three["client_out"][last])


def _sim(**kw):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    d = dict(comm_round=6, total_train_iteration=4, compression="eftopk", topk_ratio=0.2)
    d.update(kw)
    return DriftSim(make_args(**d), device="cuda", sink=MetricsSink())


def test_round_graph_replay_matches_non_graph_path_and_building_keeps_the_residual():
    def make():
        sim = _sim(client_num_per_round=3)
        for t in range(2):
            sim.run_time_step(t, rounds=4)
        sim.begin_time_step(2)
        sim.run_rounds(1)
        sim.args.rounds_per_launch = 1
        return sim

    a, b = make(), make()
    r0 = a.clients.ef_res.clone()
    assert bool((r0 != 0).any())
    ha, hb = a.make_host_round_inputs(), b.make_host_round_inputs()
    a._build_round_graph(ha)
    assert torch.equal(a.clients.ef_res, r0)   # the warm-up launch ran on a snapshot
    a._graph = None
    for _ in range(4):
        ra = a.run_round(ha, use_graph=True)
        rb = b.run_round(hb, use_graph=False)
        for k in ("train_acc", "train_loss", "test_acc", "test_loss"):
            assert abs(ra[k] - rb[k]) < 1e-5, (k, ra, rb)
    assert torch.equal(a.bank.theta, b.bank.theta) and torch.equal(a.clients.ef_res, b.clients.ef_res)


def _generic_sparsified(kw, env=None, rho=0.05):
    """One round of time step 0 on the generic executor with eftopk: the arena the round aggregated must be the oracle
    applied to the raw arena training left (bit for bit: K18 is exact), the residual likewise, and θ their weighted mean."""
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        d = dict(compression="eftopk", topk_ratio=rho)
        d.update(kw)
        sim = DriftSim(make_args(**d), device="cuda", sink=MetricsSink())
        sim.algo.fused_ok = lambda: False
        sim.begin_time_step(0)
        raw = []
        real = ops.eftopk_slots_

        def spy(rows, theta, residual, n, *a):
            raw.append((rows.clone(), residual.clone(), n.clone()))
            return real(rows, theta, residual, n, *a)
        ops.eftopk_slots_ = spy
        try:
            theta0 = sim.bank.theta.clone()
            sim.run_rounds(1)
            torch.cuda.synchronize()
        finally:
            ops.eftopk_slots_ = real
        up, r0, n = raw[0]
        want_up, want_res = up.cpu(), r0.cpu()
        mask = None if sim.defense_mask is None else sim.defense_mask.cpu()
        ref.eftopk_slots_(want_up, theta0.cpu(), want_res, n.cpu(), sim.topk_k, mask)
        assert torch.equal(sim.clients.params.cpu(), want_up)
        assert torch.equal(sim.clients.ef_res.cpu(), want_res)
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


def test_generic_per_pair_graphs_sparsify_uploads():
    sim = _generic_sparsified(dict(model="fnn", dataset="MNIST", client_num_in_total=6, concept_num=2, concept_drift_algo="softcluster",
                                   concept_drift_algo_arg="H_A_C_1_10_0", change_points="A", sample_num=16, batch_size=8, comm_round=3,
                                   total_train_iteration=2, epochs=2))
    assert any(g.indexed and g.launches > 0 for g in sim.__dict__.get("_step_graphs", {}).values()), "per-pair graphs not used"


def test_generic_stacked_resnet_sparsifies_uploads_and_keeps_bn_buffers(monkeypatch):
    from feddrift_b200.sim import stacked
    calls = []
    real = stacked.train_pairs

    def spy(sim, pairs, *a):
        calls.append(len(pairs))
        return real(sim, pairs, *a)
    monkeypatch.setattr(stacked, "train_pairs", spy)
    sim = _generic_sparsified(dict(model="resnet18", dataset="cifar10", client_num_in_total=4, concept_num=2, concept_drift_algo="win-1",
                                   concept_drift_algo_arg="", change_points="A", sample_num=8, batch_size=8, comm_round=2,
                                   total_train_iteration=2, epochs=1, client_optimizer="sgd", lr=0.05), {"FDB_STACKED": "force"},
                              rho=0.01)
    assert calls
    assert sim.defense_mask is not None and not bool(sim.defense_mask.all())


def test_generic_lstm_sparsifies_uploads():
    from feddrift_b200.ops import lstm as fused
    n0 = fused.CALLS["bwd"]
    _generic_sparsified(dict(model="rnn", dataset="shakespeare", client_num_in_total=6, concept_num=2, concept_drift_algo="win-1",
                             concept_drift_algo_arg="", change_points="A", sample_num=32, batch_size=16, comm_round=2,
                             total_train_iteration=2, epochs=2, lr=0.05, client_optimizer="sgd", report_client=0))
    assert fused.CALLS["bwd"] > n0, "batched LSTM executor did not run"


def test_drift_sim_fused_route_runs_and_ratio_one_equals_none():
    a = _sim(topk_ratio=1.0)
    b = _sim(compression="none")
    oa, ob = a.run(), b.run()
    assert torch.equal(a.bank.theta, b.bank.theta) and oa["history"] == ob["history"]
    c = _sim(topk_ratio=0.1)
    c.run()
    assert torch.isfinite(c.bank.theta).all() and not torch.allclose(c.bank.theta, b.bank.theta)


WORKER = r'''
import os, sys, json, torch, torch.distributed as dist
sys.path.insert(0, os.environ["FDB_ROOT"])
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.parallel.symm import attach_multi_gpu, check_error
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
kw = dict(comm_round=6, total_train_iteration=3, client_num_in_total=10, compression="eftopk", topk_ratio=1.0)
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
mine = [c for c in range(10) if c % world == rank]
others = [c for c in range(10) if c % world != rank]
res_ok = bool((sim.clients.ef_res[others] == 0).all())
ok = same and res_ok and err < 1e-4 and abs(out["history"][-1]["train_acc"] - oref["history"][-1]["train_acc"]) < 0.02
print(json.dumps({"rank": rank, "err": err, "ranks_identical": same, "ok": bool(ok)}))
dist.destroy_process_group()
sys.exit(0 if ok else 3)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_gpu_fused_with_eftopk_matches_single_gpu(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, FDB_ROOT=root, PYTHONFAULTHANDLER="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29547", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
