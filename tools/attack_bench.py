"""Simulated Byzantine clients on the GPU: (1) K22 (``ops.attack_slots_``) for every attack type on a config-2-sized upload
arena (fnn 3-6-2 rows, 100 clients × 4 slots) and a config-4-sized one (ResNet-18 rows, 32 clients × 2 slots), a quarter
of the clients attacking, timed with CUDA events over many launches, with the bytes each moves per launch (from the shapes)
over the time against the H100 SXM data-sheet 3.35 TB/s: sign_flip / gaussian read and write the attacker rows and read θ
once per attacker row; alie reads the honest rows twice (μ, then σ) and writes the attacker rows, ipm reads them once
and θ once; (2) config 2 rounds/s on the fused kernel without an attack and with 20 sign_flip clients, alternated in one
process.  Prints one JSON line per measurement, each with the card name and its power limit read in the same run.

    python tools/attack_bench.py [--launches 20] [--reps 5] [--rounds 40]
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
from feddrift_b200.ops import reference as ref  # noqa: E402
from feddrift_b200.parallel.arena import ModelBank  # noqa: E402
from feddrift_b200.sim import DriftSim, make_args  # noqa: E402
from feddrift_b200.utils.metrics import MetricsSink  # noqa: E402
from krum_bench import _time  # noqa: E402
from qsgd_bench import HBM_BPS, card  # noqa: E402

KINDS = ("sign_flip", "gaussian", "alie", "ipm")


def _moved(kind, C, A, M, P):
    row = M * P * 4
    if kind in ("sign_flip", "gaussian"):
        return A * row * 3                         # read x and θ, write x
    if kind == "alie":
        return 2 * (C - A) * row + A * row         # μ pass and σ pass over the honest rows, crafted rows written
    return (C - A) * row + M * P * 4 + A * row     # ipm: honest rows and θ read once, crafted rows written


def bench_k22(launches: int):
    dev = torch.device("cuda")
    out = []
    arenas = {"cfg2 fnn 3-6-2": (100, 4, ref.mlp_param_count("fnn", 3, 6, 2)),
              "cfg4 resnet18": (32, 2, ModelBank(create_model("resnet18", 10, 3, small_input=True), 1, dev).P)}
    for arena, (C, M, P) in arenas.items():
        g = torch.Generator(device=dev).manual_seed(0)
        theta = torch.randn(M, P, generator=g, device=dev)
        base = theta[None] + 0.01 * torch.randn(C, M, P, generator=g, device=dev)
        up = base.clone()
        n = torch.ones(C, M, device=dev)
        A = C // 4
        att = ref.attacker_clients(C, A, 0).to(dev)
        for kind in KINDS:
            def fn():
                ops.attack_slots_(up, theta, n, att, kind, 1.0, None, 1)
            times = _time(fn, launches)
            med = times[len(times) // 2]
            moved = _moved(kind, C, A, M, P)
            out.append({"what": "K22 attack_slots", "kind": kind, "arena_name": arena, "arena": [C, M, P], "attackers": A,
                        "launches": launches, "median_ms": med * 1e3, "min_ms": times[0] * 1e3, "max_ms": times[-1] * 1e3,
                        "bytes_moved": moved, "achieved_TBps": moved / med / 1e12, "share_of_3.35TBps": moved / med / HBM_BPS})
            up.copy_(base)
    return out


def bench_cfg2(reps: int, rounds: int):
    variants = {"none": {}, "sign_flip a=20": dict(attack_type="sign_flip", attack_clients=20, attack_scale=1.0)}
    sims = {}
    for name, extra in variants.items():
        kw = dict(CONFIGS["cfg2_sea_fnn_100clients_feddrift"])
        kw.update(total_train_iteration=2, epochs=5, lr=0.01, report_client=0, rounds_per_launch=rounds, **extra)
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.run_time_step(0, rounds=1)
        sim.begin_time_step(1)
        sim.run_rounds(2)   # warm-up
        sims[name] = sim
    torch.cuda.synchronize()
    res = {k: [] for k in variants}
    for _ in range(reps):
        for name, sim in sims.items():
            t0 = time.perf_counter()
            sim.run_rounds(rounds)
            torch.cuda.synchronize()
            res[name].append(rounds / (time.perf_counter() - t0))
    out = {"what": "cfg2 rounds/s", "rounds_per_rep": rounds, "reps": reps,
           "fused_kernel": {k: bool(s._use_fused()) for k, s in sims.items()}}
    for name in variants:
        v = sorted(res[name])
        out[name] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=40)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "attack_bench needs a GPU"
    info = card()
    for r in bench_k22(a.launches):
        print(json.dumps(dict(r, **info)), flush=True)
    print(json.dumps(dict(bench_cfg2(a.reps, a.rounds), **info)), flush=True)


if __name__ == "__main__":
    main()
