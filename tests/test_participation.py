"""Partial client participation (``client_num_per_round < client_num_in_total``) on the CPU: the selection rule against the
reference's recorded sets, the round oracle's semantics, and the device engine's fused-reference and generic paths."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from feddrift_b200.ops import reference as ref
from feddrift_b200.sim import DriftSim, make_args
from feddrift_b200.sim.sampling import sample_clients
from feddrift_b200.utils.metrics import MetricsSink
from test_gpu_small_round import make_state

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "client_sampling.json")   # tools/record_client_sampling.py


def _table(rows, C, K):
    tab = torch.zeros(rows, C, dtype=torch.bool)
    for r in range(rows):
        tab[r, torch.from_numpy(sample_clients(r, C, K))] = True
    return tab


def test_sample_clients_matches_reference_and_facade():
    from feddrift_b200.drift.fedavg_ens import _BaseAggregator
    with open(GOLDEN) as fh:
        cases = json.load(fh)["cases"]
    assert {(c["client_num_in_total"], c["client_num_per_round"]) for c in cases} == {(10, 3), (100, 10), (7, 9)}
    state = np.random.get_state()
    try:
        for case in cases:
            C, K = case["client_num_in_total"], case["client_num_per_round"]
            assert len(case["rounds"]) == 200
            for r, want in enumerate(case["rounds"]):
                got = sample_clients(r, C, K)
                assert got.tolist() == want, (C, K, r)
                assert sorted(int(c) for c in _BaseAggregator.client_sampling(None, r, C, K)) == sorted(want), (C, K, r)
    finally:
        np.random.set_state(state)


def test_sample_clients_leaves_global_rng_alone():
    np.random.seed(5)
    a = np.random.rand()
    np.random.seed(5)
    sample_clients(3, 10, 3)
    assert np.random.rand() == a


def _run_oracle(st, rounds, table=None):
    st = copy.deepcopy(st)
    if table is not None:
        st["participation"] = table
    out = ref.fed_round_small(st, rounds)
    return st, out


def test_all_ones_table_is_bit_identical_to_no_table():
    st = make_state(C=6, S=40, epochs=2)
    a, oa = _run_oracle(st, 2)
    b, ob = _run_oracle(st, 2, torch.ones(3, 6, dtype=torch.uint8))
    for k in ("theta", "opt_m", "opt_v", "opt_vmax", "opt_step", "W"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(oa["metrics"], ob["metrics"])


def test_non_participants_and_empty_clusters_are_untouched():
    C = 8
    st = make_state(C=C, S=40, epochs=2)
    # clients 1 and 5 never take part; client 5 is the only member of cluster 2 at t_cur (make_state's plan)
    table = torch.ones(3, C, dtype=torch.bool)
    table[:, [1, 5]] = False
    table[1, [0, 2, 3]] = False
    theta0 = st["theta"].clone()
    out_st, out = _run_oracle(st, 3, table)
    for c in (1, 5):
        for k in ("opt_m", "opt_v", "opt_vmax", "opt_step"):
            assert torch.equal(out_st[k][c], st[k][c]), (c, k)
    assert torch.equal(out_st["theta"][2], theta0[2])
    assert not torch.equal(out_st["theta"][0], theta0[0])
    assert (out_st["opt_step"][0] > 0).any() and (out_st["opt_step"][4] > 0).any()
    # every client is still evaluated, participant or not
    assert (out["metrics"][..., 1] > 0).all() and (out["metrics"][..., 3] > 0).all()
    assert torch.equal(out["counts"], ref.fed_round_small(copy.deepcopy(st), 1)["counts"])


def test_single_participant_cluster_equals_its_local_model():
    C = 6
    st = make_state(C=C, S=40, epochs=3)
    c0 = 3
    st["W"][:, :, c0] = 0
    st["W"][:, 0, c0] = 1   # c0 trains cluster 0 only; cluster 0 has other members too
    table = torch.zeros(1, C, dtype=torch.bool)
    table[0, c0] = True
    got, _ = _run_oracle(st, 1, table)
    # the same round with c0 as cluster 0's only member by plan: FedAvg over one client is that client's local model
    solo = copy.deepcopy(st)
    solo["W"][:, :, [c for c in range(C) if c != c0]] = 0
    want, _ = _run_oracle(solo, 1)
    assert not torch.equal(got["theta"][0], st["theta"][0])
    assert torch.equal(got["theta"], want["theta"])
    assert torch.equal(got["opt_step"], want["opt_step"])


def _sea_args(**kw):
    d = dict(client_num_in_total=10, client_num_per_round=3, comm_round=4, total_train_iteration=3, sample_num=40, epochs=2)
    d.update(kw)
    return make_args(**d)


def _check_rounds_follow_table(sim, rounds, generic):
    for r in range(rounds):
        step0 = sim.clients.step.clone()
        sim.run_rounds(1)
        row = sim.participants(r)
        changed = (sim.clients.step != step0).any(dim=1).numpy()
        assert changed.any() and not (changed & ~row).any(), (r, changed, row)
        if generic:
            trained = (sim.clients.n > 0).any(dim=1).numpy()
            assert trained.any() and not (trained & ~row).any(), (r, trained, row)


def test_drift_sim_fused_reference_path_samples_clients():
    sink = MetricsSink()
    sim = DriftSim(_sea_args(), device="cpu", sink=sink)
    assert sim.participation is not None and sim.participation.shape == (4, 10)
    assert (sim.participation.sum(1) == 3).all()
    sim.begin_time_step(0)
    _check_rounds_follow_table(sim, 4, generic=False)
    sim.end_time_step()
    out = sim.run(start_iteration=1)
    assert len(out["history"]) >= 3
    for c in range(10):
        assert len(sink.series(f"Train/Acc-CL-{c}")) >= 3 and len(sink.series(f"Test/Acc-CL-{c}")) >= 3


def test_drift_sim_generic_path_samples_clients():
    sink = MetricsSink()
    sim = DriftSim(_sea_args(), device="cpu", sink=sink)
    sim.algo.fused_ok = lambda: False
    sim.begin_time_step(0)
    _check_rounds_follow_table(sim, 4, generic=True)
    sim.end_time_step()
    ref_sim = DriftSim(_sea_args(), device="cpu", sink=MetricsSink())
    ref_sim.run(end_iteration=1)
    assert torch.allclose(sim.bank.theta, ref_sim.bank.theta, rtol=1e-4, atol=1e-5)   # same plan semantics as the oracle


def test_drift_sim_cnn_generic_path_samples_clients():
    sink = MetricsSink()
    sim = DriftSim(make_args(model="cnn", dataset="MNIST", client_num_in_total=5, client_num_per_round=2, sample_num=12,
                             batch_size=4, comm_round=3, total_train_iteration=2, concept_drift_algo="win-1", epochs=1),
                   device="cpu", sink=sink)
    sim.begin_time_step(0)
    _check_rounds_follow_table(sim, 3, generic=True)
    sim.end_time_step()
    sim.run(start_iteration=1)
    for c in range(5):
        assert len(sink.series(f"Test/Acc-CL-{c}")) >= 1


def test_full_participation_builds_no_table_and_bad_k_raises():
    assert DriftSim(_sea_args(client_num_per_round=10), device="cpu", sink=MetricsSink()).participation is None
    assert DriftSim(_sea_args(client_num_per_round=12), device="cpu", sink=MetricsSink()).participation is None
    with pytest.raises(ValueError):
        DriftSim(_sea_args(client_num_per_round=0), device="cpu", sink=MetricsSink())


def test_clusterfl_split_keeps_non_participants_on_model_zero():
    sim = DriftSim(_sea_args(concept_drift_algo="clusterfl", concept_drift_algo_arg="win-1", concept_num=2, client_num_in_total=8,
                             client_num_per_round=4), device="cpu", sink=MetricsSink())
    sim.algo.split_round = 2
    sim.run_time_step(0)
    assert sim.algo.split_done
    row = sim.participants(2)
    assert (sim.algo.assign[~row] == 0).all()
    assert (sim.algo.assign[row] == 1).any()
