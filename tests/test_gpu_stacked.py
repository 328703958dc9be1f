"""Pair-stacked executor on the GPU: the stacked path equals the per-pair path (SGD, dropout-free CNN; see tests/test_stacked.py
for the CPU equivalence proofs)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(stacked: str, rounds: int = 3):
    from feddrift_b200.sim import DriftSim, make_args
    from feddrift_b200.utils.metrics import MetricsSink
    os.environ["FDB_STACKED"] = stacked
    try:
        a = make_args(model="cnn", dataset="MNIST", client_num_in_total=6, client_num_per_round=6, concept_drift_algo="win-1",
                      concept_drift_algo_arg="", concept_num=2, change_points="A", sample_num=16, batch_size=8, comm_round=rounds,
                      total_train_iteration=2, epochs=2, lr=0.05, report_client=0, client_optimizer="sgd")
        sim = DriftSim(a, device="cuda", sink=MetricsSink())
        for mod in (sim.bank.template.dropout_1, sim.bank.template.dropout_2):
            mod.p = 0.0
        sim.run_time_step(0, rounds=rounds)
        torch.cuda.synchronize()
        return sim.bank.theta.clone()
    finally:
        os.environ.pop("FDB_STACKED", None)


def test_stacked_equals_per_pair():
    th_stacked = _run("force")
    th_pair = _run("0")
    scale = th_pair.abs().max().item()
    assert (th_stacked - th_pair).abs().max().item() < 2e-2 * scale     # bf16 tensor-core operands on both sides, different summation orders
