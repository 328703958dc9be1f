"""Top-k sparsification with error feedback on the GPU: (1) the K18 kernel (``ops.eftopk_slots_``) on a config-4-sized upload
arena (ResNet-18 rows, 32 clients × 2 slots, BatchNorm mask) at ρ ∈ {0.001, 0.01, 0.1}, timed with CUDA events over many
launches, with the bytes its passes move per launch over the kernel time against the H100 SXM data-sheet 3.35 TB/s; (2)
config 2 rounds/s with ``--compression none`` and ``eftopk`` (ρ = 0.25), alternated in one process.  Prints one JSON line
per measurement, each with the card name and its power limit read in the same run.

    python tools/eftopk_bench.py [--launches 20] [--reps 5]
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
from feddrift_b200.models import utils as mutils  # noqa: E402
from feddrift_b200.models.utils import create_model  # noqa: E402
from feddrift_b200.ops import reference as ref  # noqa: E402
from feddrift_b200.parallel.arena import ModelBank  # noqa: E402
from feddrift_b200.sim import DriftSim, make_args  # noqa: E402
from feddrift_b200.utils.metrics import MetricsSink  # noqa: E402
from qsgd_bench import HBM_BPS, card  # noqa: E402


def bench_k18(launches: int, rhos=(0.001, 0.01, 0.1)):
    dev = torch.device("cuda")
    bank = ModelBank(create_model("resnet18", 10, 3, small_input=True), 2, dev)
    P, M, C = bank.P, 2, 32
    mask = mutils.weight_param_mask(bank.spec)[:P].to(dev)
    n_train = int(mask.sum())
    g = torch.Generator(device=dev).manual_seed(0)
    bank.theta.copy_(torch.randn(M, bank.theta.shape[1], generator=g, device=dev))
    raw = bank.theta[None, :, :P] + 0.01 * torch.randn(C, M, P, generator=g, device=dev)
    res0 = 0.001 * torch.randn(C, M, P, generator=g, device=dev)
    rows, res = raw.clone(), res0.clone()
    n = torch.ones(C, M, device=dev)
    R = C * M
    out = []
    for rho in rhos:
        k = ref.topk_k(rho, n_train)
        for _ in range(3):   # warm-up
            rows.copy_(raw)
            res.copy_(res0)
            ops.eftopk_slots_(rows, bank.theta, res, n, k, mask)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * launches)]
        for i in range(launches):
            rows.copy_(raw)   # every launch sparsifies the raw arena against the same residual
            res.copy_(res0)
            ev[2 * i].record()
            ops.eftopk_slots_(rows, bank.theta, res, n, k, mask)
            ev[2 * i + 1].record()
        torch.cuda.synchronize()
        times = sorted(ev[2 * i].elapsed_time(ev[2 * i + 1]) * 1e-3 for i in range(launches))
        med = times[len(times) // 2]
        # the three histogram passes read x, θ, e and the mask byte; the apply pass reads them and writes x, e.  The tie pass
        # (one more read) only runs for rows whose threshold key is shared by more entries than it keeps, so it is not counted
        moved = R * P * (13 * 4 + 8)
        minimal = R * P * 20   # x, θ, e read once, x, e written once
        out.append({"what": "K18 eftopk_slots", "arena": [C, M, P], "n_train": n_train, "topk_ratio": rho, "k": k,
                    "launches": launches, "median_ms": med * 1e3, "min_ms": times[0] * 1e3, "max_ms": times[-1] * 1e3,
                    "bytes_moved": moved, "achieved_TBps": moved / med / 1e12, "share_of_3.35TBps": moved / med / HBM_BPS,
                    "one_pass_bytes": minimal, "one_pass_TBps": minimal / med / 1e12})
    return out


def bench_cfg2(reps: int, rounds: int):
    sims = {}
    for comp in ("none", "eftopk"):
        kw = dict(CONFIGS["cfg2_sea_fnn_100clients_feddrift"])
        kw.update(total_train_iteration=2, epochs=5, lr=0.01, report_client=0)
        if comp == "eftopk":
            kw.update(compression="eftopk", topk_ratio=0.25)
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.run_time_step(0, rounds=1)
        sim.begin_time_step(1)
        sim.run_rounds(2)   # warm-up
        sims[comp] = sim
    torch.cuda.synchronize()
    res = {"none": [], "eftopk": []}
    for _ in range(reps):
        for comp in ("none", "eftopk"):
            t0 = time.perf_counter()
            sims[comp].run_rounds(rounds)
            torch.cuda.synchronize()
            res[comp].append(rounds / (time.perf_counter() - t0))
    out = {"what": "cfg2 rounds/s", "rounds_per_rep": rounds, "reps": reps,
           "fused_kernel": bool(sims["eftopk"]._use_fused())}
    for comp, v in res.items():
        v = sorted(v)
        out[comp] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=40)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "eftopk_bench needs a GPU"
    info = card()
    for r in bench_k18(a.launches):
        print(json.dumps(dict(r, **info)), flush=True)
    print(json.dumps(dict(bench_cfg2(a.reps, a.rounds), **info)), flush=True)


if __name__ == "__main__":
    main()
