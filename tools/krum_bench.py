"""Multi-Krum on the GPU: (1) the K21 kernel sequence (``ops.krum_aggregate_slots_``, f = 1, m = 1 and m = 4) against K1
(mean), K19 (median) and K20 (geometric median, R = 4) on a config-4-sized upload arena (ResNet-18 rows, 32 clients × 2
slots), timed with CUDA events over many launches, with the bytes each moves per launch over the time against the H100 SXM
data-sheet 3.35 TB/s (K21: one read of the participants' rows in the distance pass, the m_eff selected rows again in the
store pass, θ written once; the fp64 pair partials are left out); (2) config 2 rounds/s with ``--aggregation_rule`` mean,
median, geometric_median and multi_krum, alternated in one process, plus the fused kernel's aggregation-phase time per
round (train end → aggregation end, from its ``timers`` stamps).  Prints one JSON line per measurement, each with the card
name and its power limit read in the same run.

    python tools/krum_bench.py [--launches 20] [--reps 5] [--rounds 40]
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
from qsgd_bench import HBM_BPS, card  # noqa: E402

ITERS = 4
RULES = {"mean": None, "median": ("median", 0.1), "geometric_median": ("geometric_median", 0.1, ITERS, 1e-6),
         "multi_krum m=1": ("multi_krum", 0.1, 1, 1), "multi_krum m=4": ("multi_krum", 0.1, 1, 4)}
KERNEL = {"mean": "K1 cluster_aggregate", "median": "K19 robust_aggregate_slots",
          "geometric_median": "K20 geomed_aggregate_slots", "multi_krum m=1": "K21 krum_aggregate_slots",
          "multi_krum m=4": "K21 krum_aggregate_slots"}
CFG2_RULES = {"mean": {}, "median": dict(aggregation_rule="median"), "geometric_median": dict(aggregation_rule="geometric_median"),
              "multi_krum": dict(aggregation_rule="multi_krum", krum_f=1, krum_m=1)}


def _time(fn, launches):
    for _ in range(3):   # warm-up
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * launches)]
    for i in range(launches):
        ev[2 * i].record()
        fn()
        ev[2 * i + 1].record()
    torch.cuda.synchronize()
    return sorted(ev[2 * i].elapsed_time(ev[2 * i + 1]) * 1e-3 for i in range(launches))


def bench_k21(launches: int):
    dev = torch.device("cuda")
    bank = ModelBank(create_model("resnet18", 10, 3, small_input=True), 2, dev)
    P, M, C = bank.P, 2, 32
    g = torch.Generator(device=dev).manual_seed(0)
    theta0 = torch.randn(M, bank.theta.shape[1], generator=g, device=dev)
    up = theta0[None, :, :P] + 0.01 * torch.randn(C, M, P, generator=g, device=dev)
    n = torch.ones(C, M, device=dev)
    out = []
    for name, rule in RULES.items():
        def fn():
            ops.cluster_aggregate_(bank.theta, up, n, None, rule)
        times = _time(fn, launches)
        med = times[len(times) // 2]
        moved = C * M * P * 4 + M * P * 4   # every upload read once, θ written once
        if name == "geometric_median":
            moved = (ITERS + 2) * C * M * P * 4 + (ITERS + 2) * M * P * 4
        elif rule is not None and rule[0] == "multi_krum":
            moved += min(rule[3], C) * M * P * 4   # the store pass reads the selected rows again
        out.append({"what": KERNEL[name], "rule": name, "arena": [C, M, P],
                    "launches": launches, "median_ms": med * 1e3, "min_ms": times[0] * 1e3, "max_ms": times[-1] * 1e3,
                    "bytes_moved": moved, "achieved_TBps": moved / med / 1e12, "share_of_3.35TBps": moved / med / HBM_BPS})
    return out


def bench_cfg2(reps: int, rounds: int):
    sims = {}
    for name, extra in CFG2_RULES.items():
        kw = dict(CONFIGS["cfg2_sea_fnn_100clients_feddrift"])
        kw.update(total_train_iteration=2, epochs=5, lr=0.01, report_client=0, rounds_per_launch=rounds, **extra)
        sim = DriftSim(make_args(**kw), device="cuda", sink=MetricsSink())
        sim.run_time_step(0, rounds=1)
        sim.begin_time_step(1)
        sim.run_rounds(2)   # warm-up
        sims[name] = sim
    torch.cuda.synchronize()
    res = {k: [] for k in CFG2_RULES}
    agg = {k: [] for k in CFG2_RULES}
    for _ in range(reps):
        for name, sim in sims.items():
            t0 = time.perf_counter()
            sim.run_rounds(rounds)
            torch.cuda.synchronize()
            res[name].append(rounds / (time.perf_counter() - t0))
    for name, sim in sims.items():   # one more block with the kernel's phase stamps on (a separate, untimed run)
        st = sim._small_state()
        st["timers"] = torch.zeros(rounds, 4, dtype=torch.int64, device="cuda")
        sim.run_rounds(rounds)
        torch.cuda.synchronize()
        t = st.pop("timers").cpu()
        t = t[t[:, 0] > 0]
        agg[name] = sorted(((t[:, 1] - t[:, 0]).double() * 1e-3).tolist())
    out = {"what": "cfg2 rounds/s", "rounds_per_rep": rounds, "reps": reps,
           "fused_kernel": {k: bool(s._use_fused()) for k, s in sims.items()}}
    for name in CFG2_RULES:
        v = sorted(res[name])
        a = agg[name]
        out[name] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1],
                     "agg_phase_us_median": a[len(a) // 2] if a else None, "agg_phase_rounds": len(a)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=40)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "krum_bench needs a GPU"
    info = card()
    for r in bench_k21(a.launches):
        print(json.dumps(dict(r, **info)), flush=True)
    print(json.dumps(dict(bench_cfg2(a.reps, a.rounds), **info)), flush=True)


if __name__ == "__main__":
    main()
