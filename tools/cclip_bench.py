"""Centered clipping on the GPU: (1) the K23 kernel sequence (``ops.cclip_aggregate_slots_``) for L = 1 and L = 3 against
K1 (mean) on a config-4-sized upload arena (ResNet-18 rows, 32 clients × 2 slots), timed with CUDA events over many launches,
with the bytes each moves per launch (K23: L + 1 reads of the participants' rows plus θ and the center's traffic) over the
time against the H100 SXM data-sheet 3.35 TB/s; (2) config 2 rounds/s with ``--aggregation_rule`` mean and centered_clip (τ
and L of ``cfg2c_sea_fnn_100clients_cclip_feddrift``), alternated in one process, on the fused round kernel.  Prints one
JSON line per measurement, each with the card name and its power limit read in the same run.

    python tools/cclip_bench.py [--launches 20] [--reps 5] [--rounds 40]
"""
import argparse
import json
import sys
import time

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
from feddrift_b200 import ops  # noqa: E402
from feddrift_b200.experiments.configs import CONFIGS  # noqa: E402
from feddrift_b200.models.utils import create_model  # noqa: E402
from feddrift_b200.parallel.arena import ModelBank  # noqa: E402
from feddrift_b200.sim import DriftSim, make_args  # noqa: E402
from feddrift_b200.utils.metrics import MetricsSink  # noqa: E402
from geomed_bench import _time  # noqa: E402
from qsgd_bench import HBM_BPS, card  # noqa: E402

CFG = CONFIGS["cfg2c_sea_fnn_100clients_cclip_feddrift"]


def k23_bytes(C: int, M: int, P: int, L: int) -> int:
    """Bytes K23 moves per launch: L + 1 reads of the rows and of θ, one write of θ, and the center's 1 + 2L reads and writes
    (pass 1 reads it, every later pass reads and rewrites it)."""
    return 4 * ((L + 1) * C * M * P + (L + 1) * M * P + M * P + (1 + 2 * L) * M * P)


def bench_k23(launches: int):
    dev = torch.device("cuda")
    bank = ModelBank(create_model("resnet18", 10, 3, small_input=True), 2, dev)
    P, M, C = bank.P, 2, 32
    g = torch.Generator(device=dev).manual_seed(0)
    theta0 = torch.randn(M, bank.theta.shape[1], generator=g, device=dev)
    bank.theta.copy_(theta0[:, :P])
    up = theta0[None, :, :P] + 0.01 * torch.randn(C, M, P, generator=g, device=dev)
    n = torch.ones(C, M, device=dev)
    center = torch.zeros(M, P, device=dev)
    tau = 0.5 * float(torch.linalg.vector_norm(up[0, 0] - theta0[0, :P]))   # clips every row
    out = []
    for name, rule in (("mean", None), ("centered_clip L=1", ("centered_clip", 0.1, tau, 1)),
                       ("centered_clip L=3", ("centered_clip", 0.1, tau, 3))):
        def fn():   # θ and the center move from launch to launch; the work per launch does not depend on them
            ops.cluster_aggregate_(bank.theta, up, n, None, rule, center=center)

        times = _time(fn, launches)
        med = times[len(times) // 2]
        moved = C * M * P * 4 + M * P * 4 if rule is None else k23_bytes(C, M, P, rule[3])
        out.append({"what": "K1 cluster_aggregate" if rule is None else "K23 cclip_aggregate_slots", "rule": name,
                    "arena": [C, M, P], "launches": launches, "median_ms": med * 1e3, "min_ms": times[0] * 1e3,
                    "max_ms": times[-1] * 1e3, "bytes_moved": moved,
                    "achieved_TBps": moved / med / 1e12, "share_of_3.35TBps": moved / med / HBM_BPS})
    return out


def bench_cfg2(reps: int, rounds: int):
    sims = {}
    for name in ("mean", "centered_clip"):
        kw = dict(CONFIGS["cfg2_sea_fnn_100clients_feddrift"])
        kw.update(total_train_iteration=2, epochs=5, lr=0.01, report_client=0, rounds_per_launch=rounds)
        if name != "mean":
            kw.update(aggregation_rule=name, cclip_tau=CFG["cclip_tau"], cclip_iters=CFG["cclip_iters"])
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.run_time_step(0, rounds=1)
        sim.begin_time_step(1)
        sim.run_rounds(2)   # warm-up
        sims[name] = sim
    torch.cuda.synchronize()
    res = {k: [] for k in sims}
    for _ in range(reps):
        for name, sim in sims.items():
            t0 = time.perf_counter()
            sim.run_rounds(rounds)
            torch.cuda.synchronize()
            res[name].append(rounds / (time.perf_counter() - t0))
    out = {"what": "cfg2 rounds/s", "rounds_per_rep": rounds, "reps": reps, "cclip_tau": CFG["cclip_tau"],
           "cclip_iters": CFG["cclip_iters"], "fused_kernel": {k: bool(s._use_fused()) for k, s in sims.items()}}
    for name in sims:
        v = sorted(res[name])
        out[name] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=40)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "cclip_bench needs a GPU"
    info = card()
    for r in bench_k23(a.launches):
        print(json.dumps(dict(r, **info)), flush=True)
    print(json.dumps(dict(bench_cfg2(a.reps, a.rounds), **info)), flush=True)


if __name__ == "__main__":
    main()
