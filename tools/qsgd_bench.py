"""QSGD upload compression on the GPU: (1) the K17 kernel (``ops.qsgd_slots_``) on a config-4-sized upload arena (ResNet-18
rows, 32 clients × 2 slots, BatchNorm mask) timed with CUDA events over many launches, with the bytes its two passes move
per launch over the kernel time against the H100 SXM data-sheet 3.35 TB/s; (2) config 2 rounds/s with ``--compression none``
and ``qsgd`` (s = 4), alternated in one process.  Prints one JSON line per measurement, each with the card name and its power
limit read in the same run.

    python tools/qsgd_bench.py [--launches 50] [--reps 5]
"""
import argparse
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
from feddrift_b200 import ops  # noqa: E402
from feddrift_b200.experiments.configs import CONFIGS  # noqa: E402
from feddrift_b200.models import utils as mutils  # noqa: E402
from feddrift_b200.models.utils import create_model  # noqa: E402
from feddrift_b200.parallel.arena import ModelBank  # noqa: E402
from feddrift_b200.sim import DriftSim, make_args  # noqa: E402
from feddrift_b200.utils.metrics import MetricsSink  # noqa: E402

HBM_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, plim = torch.cuda.get_device_name(), "unknown"
    return {"gpu": name, "power_limit": plim}


def bench_k17(launches: int, level: int = 4, bucket: int = 512):
    dev = torch.device("cuda")
    bank = ModelBank(create_model("resnet18", 10, 3, small_input=True), 2, dev)
    P, M, C = bank.P, 2, 32
    mask = mutils.weight_param_mask(bank.spec)[:P].to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    bank.theta.copy_(torch.randn(M, bank.theta.shape[1], generator=g, device=dev))
    raw = bank.theta[None, :, :P] + 0.01 * torch.randn(C, M, P, generator=g, device=dev)
    rows = raw.clone()
    n = torch.ones(C, M, device=dev)
    for _ in range(3):   # warm-up
        rows.copy_(raw)
        ops.qsgd_slots_(rows, bank.theta, n, level, bucket, mask, 1)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * launches)]
    times = []
    for i in range(launches):
        rows.copy_(raw)   # every launch quantizes the raw arena (not already-quantized rows)
        ev[2 * i].record()
        ops.qsgd_slots_(rows, bank.theta, n, level, bucket, mask, i)
        ev[2 * i + 1].record()
    torch.cuda.synchronize()
    times = sorted(ev[2 * i].elapsed_time(ev[2 * i + 1]) * 1e-3 for i in range(launches))
    med = times[len(times) // 2]
    R = C * M
    # pass 1 reads x and θ, pass 2 reads x and θ and writes x; each pass reads the mask byte; the scratch is R·⌈P/b⌉ words
    moved = R * P * (4 + 4 + 1) + R * P * (4 + 4 + 4 + 1) + 2 * R * ((P + bucket - 1) // bucket) * 4
    minimal = R * P * 12   # x read, θ read, x written once
    return {"what": "K17 qsgd_slots", "arena": [C, M, P], "level": level, "bucket": bucket, "launches": launches,
            "median_ms": med * 1e3, "min_ms": times[0] * 1e3, "max_ms": times[-1] * 1e3,
            "bytes_moved": moved, "achieved_TBps": moved / med / 1e12, "share_of_3.35TBps": moved / med / HBM_BPS,
            "one_pass_bytes": minimal, "one_pass_TBps": minimal / med / 1e12}


def bench_cfg2(reps: int, rounds: int):
    sims = {}
    for comp in ("none", "qsgd"):
        kw = dict(CONFIGS["cfg2_sea_fnn_100clients_feddrift"])
        kw.update(total_train_iteration=2, epochs=5, lr=0.01, report_client=0)
        if comp == "qsgd":
            kw.update(compression="qsgd", quantize_level=4, quantize_bucket=512)
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.run_time_step(0, rounds=1)
        sim.begin_time_step(1)
        sim.run_rounds(2)   # warm-up
        sims[comp] = sim
    torch.cuda.synchronize()
    res = {"none": [], "qsgd": []}
    for _ in range(reps):
        for comp in ("none", "qsgd"):
            t0 = time.perf_counter()
            sims[comp].run_rounds(rounds)
            torch.cuda.synchronize()
            res[comp].append(rounds / (time.perf_counter() - t0))
    out = {"what": "cfg2 rounds/s", "rounds_per_rep": rounds, "reps": reps,
           "fused_kernel": bool(sims["qsgd"]._use_fused())}
    for comp, v in res.items():
        v = sorted(v)
        out[comp] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=40)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "qsgd_bench needs a GPU"
    info = card()
    print(json.dumps(dict(bench_k17(a.launches), **info)), flush=True)
    print(json.dumps(dict(bench_cfg2(a.reps, a.rounds), **info)), flush=True)


if __name__ == "__main__":
    main()
