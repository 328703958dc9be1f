"""Symmetric-memory plumbing for the multi-GPU fused round kernel.

Every rank allocates one identically-shaped buffer through ``torch.distributed._symmetric_memory`` (CUDA VMM +
fabric handles under the hood); after the rendezvous each rank holds a device pointer to EVERY peer's buffer, so
the kernel can store partial sums straight into the peers' inboxes over NVLink — no NCCL call on the
aggregate/broadcast path (BASELINE.json north star).  Both areas use the LL ("low latency") format: payload and round
epoch travel in the same 8- / 16-byte store, so there are no fences, no flag words and no round trips.

Layout of the per-rank buffer:   inbox  uint2 {value, epoch}             [2 (parity)] [world] [M·P]
                                 staging uint4 {corr, epoch, loss, epoch} [max_rounds] [C] [2 (train | test)]
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.distributed as dist


def _rendezvous(numel: int, device) -> Dict:
    import torch.distributed._symmetric_memory as symm_mem
    buf = symm_mem.empty(numel, dtype=torch.float32, device=device)
    buf.zero_()
    hdl = symm_mem.rendezvous(buf, group=dist.group.WORLD.group_name)
    return {"buf": buf, "hdl": hdl, "ptrs": [int(p) for p in hdl.buffer_ptrs]}


def attach_multi_gpu(sim, world: int, rank: int) -> None:
    """Give ``sim`` the symmetric inbox / metrics-staging pointers; clients are then sharded ``c % world == rank``."""
    if getattr(sim.bank, "server_opt", None) is not None:
        raise ValueError("a server optimizer (--server_optimizer) is single-GPU only: attach_multi_gpu refuses it")
    if getattr(sim, "agg_rule", None) is not None:
        raise ValueError("a robust aggregation rule (--aggregation_rule) is single-GPU only: attach_multi_gpu refuses it")
    if getattr(sim, "attack", None) is not None:
        raise ValueError("a simulated attack (--attack_type) is single-GPU only: attach_multi_gpu refuses it")
    MP = sim.M * sim.bank.P
    inbox_floats = 2 * (2 * world * MP)                      # 8-byte LL words
    inbox_floats = (inbox_floats + 31) // 32 * 32            # staging area starts on its own 128-byte line
    max_rounds = int(getattr(sim.args, "max_rounds_per_launch", 0) or max(sim.args.comm_round, 256))
    staging_floats = 4 * (max_rounds * sim.C * 2)            # 16-byte LL words
    r = _rendezvous(inbox_floats + staging_floats, sim.device)
    base = r["ptrs"]
    sim.multi = {
        "world": world, "rank": rank, "flag_base": 0,
        "inbox_ptrs": base, "metrics_ptrs": [p + 4 * inbox_floats for p in base], "metrics_rounds": max_rounds,
        # pinned + device-mapped: the kernel raises it with a system-scope atomic on a spin timeout and the host can test
        # it after any stream sync without another device round trip
        "error_flag": torch.zeros(1, dtype=torch.int32).pin_memory(),
        "_keepalive": r,
    }
    sim.multi["error_np"] = sim.multi["error_flag"].numpy()   # zero-overhead host view for the per-round check
    torch.cuda.synchronize()
    dist.barrier()


def check_error(sim) -> None:
    """Raise if the fused kernel gave up waiting for a peer (call after a stream sync; reads pinned host memory)."""
    m = getattr(sim, "multi", None)
    if m is not None and m["error_np"][0] != 0:
        code = int(m["error_np"][0])
        raise RuntimeError(f"fed_round_small: rank {m['rank']} gave up waiting for a peer ("
                           f"{'aggregation inbox' if code == 1 else 'metrics rows'} never arrived within the spin timeout); "
                           "the cluster models were NOT updated from the incomplete inbox")
