"""Python side of the fused persistent round kernel (``csrc/fed_round_small.cu``): packs the state dict
into the launch arguments, keeps the metrics on device, and (multi-GPU) wires the symmetric inbox/flag
buffers.  One call == one kernel launch == ``rounds`` complete FL rounds."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _ext
from .reference import ATTACK_ID, attack_params, attack_table

KIND_ID = {"lr": 0, "fnn": 1}
MODE_ID = {"pool": 0, "time": 1, "index": 2}
AGG_RULE_ID = {"mean": 0, "median": 1, "trimmed_mean": 2, "geometric_median": 3, "multi_krum": 4, "centered_clip": 5}
LAUNCH_COUNT = {"fed_round_small": 0}


def supported(kind: str, din: int, hid: int, dout: int) -> bool:
    ext = _ext.load()
    return ext is not None and bool(ext.fed_round_small_supported(KIND_ID[kind], din, hid, dout))


def fits(kind: str, din: int, hid: int, dout: int, C: int, M: int, t_cur: int, server_opt: bool = False,
         robust: bool = False, rule: Optional[str] = None, attack: Optional[str] = None) -> bool:
    """True when the fused kernel can run this federation at time step ``t_cur`` (instantiated MLP shape, ``t_cur`` below
    the kernel's plan-table limit, shared-memory layout — plus the ``[2, M, P]`` server optimizer state when
    ``server_opt`` — within 227 KB, and with a ``robust`` aggregation rule 2·C ≤ 33·P for the ranking scratch; ``rule``
    'geometric_median' (implies ``robust``) also needs a slot's C uploads and weights in the CTA's gradient buffers,
    'multi_krum' a slot's C uploads with per-warp distance rows in them, and 'centered_clip' the geometric median's room);
    the ``attack`` types 'alie' and 'ipm' need statistics over every upload of a slot before the defense, so they never fit
    ('sign_flip' and 'gaussian' run in the publish step); otherwise route to the generic executor."""
    ext = _ext.load()
    if ext is None:
        return True   # CPU reference has no such limits
    rid = AGG_RULE_ID[rule] if rule not in (None, "mean") else (1 if robust else 0)
    return bool(ext.fed_round_small_fits(KIND_ID[kind], din, hid, dout, int(C), int(M), int(t_cur), bool(server_opt), rid,
                                         ATTACK_ID[attack or "none"]))


def spin_timeout_ms(st: Dict) -> int:
    """Cross-GPU spin bound: generous by default (a peer may legitimately be busy for seconds in host-side clustering or
    a CUDA-graph build); ``FDB_SPIN_TIMEOUT_MS`` / ``st['spin_timeout_ms']`` override it."""
    import os
    return int(st.get("spin_timeout_ms") or os.environ.get("FDB_SPIN_TIMEOUT_MS", 60000))


def _i32(t: Optional[torch.Tensor], dev) -> Optional[torch.Tensor]:
    if t is None:
        return None
    return t.to(device=dev, dtype=torch.int32).contiguous()


def _f32(t: Optional[torch.Tensor], dev) -> Optional[torch.Tensor]:
    if t is None:
        return None
    return t.to(device=dev, dtype=torch.float32).contiguous()


def prepare(st: Dict) -> Dict:
    """Build (once per time step) the device views the kernel reads: fp32 X, int32 Y / nsamp / index tables."""
    cache = st.setdefault("_native", {})
    if not cache:
        theta = st["theta"]
        dev = theta.device
        X = st["X"]
        T1, C, S = X.shape[0], X.shape[1], X.shape[2]
        cache["X"] = X.reshape(T1, C, S, -1).to(torch.float32).contiguous()
        cache["Y"] = _i32(st["Y"], dev)
        cache["nsamp"] = _i32(st["nsamp"], dev)
        cache["train_index"] = _i32(st.get("train_index"), dev)
        cache["train_count"] = _i32(st.get("train_count"), dev)
        cache["feat_mask"] = _f32(st.get("feat_mask"), dev)
        cache["eval_train_model"] = _i32(st.get("eval_train_model"), dev)
        cache["eval_test_model"] = _i32(st.get("eval_test_model"), dev)
        part = st.get("participation")   # [rows, C] bool/uint8 or None (everyone takes part)
        cache["participation"] = None if part is None else part.to(device=dev, dtype=torch.uint8).contiguous()
        # launch shape hints: warps per pair from the mini-batch size, cluster size from the active pair count (counted
        # as if every client took part: an upper bound when clients are sampled)
        B, t = int(st["batch_size"]), int(st["t_cur"])
        bmax = min(B, int(cache["nsamp"].max()))
        cache["wpp"] = 4 if bmax > 64 else (2 if bmax > 32 else 1)
        P = theta.shape[1]
        nwarps = 16 if P <= 24 else (12 if P <= 40 else 8)
        groups = max(1, nwarps // cache["wpp"])
        if st.get("recluster_hard"):
            npairs = C * theta.shape[0]
        elif st.get("sample_mode", "pool") == "index":
            npairs = int((cache["train_count"] > 0).sum())
        else:
            Wc = st["W"][: t + 1].detach().float().cpu()
            active = (Wc[t] != 0).any(dim=1)
            npairs = int(((Wc.sum(0) > 0) & active[:, None]).sum())
        mg = st.get("multi_gpu")
        if mg:
            npairs = -(-npairs // int(mg["world"]))
        G = 1
        while G < 8 and G * groups < npairs:
            G *= 2
        cache["cluster"] = G
        cache["counts"] = torch.stack(
            [cache["nsamp"][st["t_cur"]],
             cache["nsamp"][st["t_cur"] + 1] if st["t_cur"] + 1 < T1 else torch.zeros_like(cache["nsamp"][0])],
            dim=1).float()
    return cache


def run_native(st: Dict, rounds: int, metrics_out: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    ext = _ext.load(required=True)
    theta = st["theta"]
    dev = theta.device
    X, W = st["X"], st["W"]
    T1, C, S = X.shape[0], X.shape[1], X.shape[2]
    M = theta.shape[0]
    cache = prepare(st)
    if not (W.is_cuda and W.dtype == torch.float32 and W.is_contiguous()):
        st["W"] = W = W.to(device=dev, dtype=torch.float32).contiguous()
    ens_w = _f32(st.get("ens_w"), dev)
    use_adam = st.get("optimizer", "adam") != "sgd"
    if metrics_out is None:
        metrics_out = torch.zeros(rounds, C, 4, dtype=torch.float32, device=dev)
    lr = st["lr"]
    lr_dev = lr if isinstance(lr, torch.Tensor) else None
    Lmax = int(cache["train_index"].shape[2]) if cache["train_index"] is not None else 0
    mg = st.get("multi_gpu")  # dict(world, rank, inbox_ptrs, metrics_ptrs, flag_base, error_flag)
    world = int(mg["world"]) if mg else 1
    icfg = [T1, C, S, M, Lmax, int(st["batch_size"]), int(st["epochs"]), int(st["t_cur"]), int(rounds), int(st["round0"]),
            int(st["seed"]) & 0xFFFFFFFF, int(use_adam), MODE_ID[st.get("sample_mode", "pool")],
            1 if st.get("n_mode", "batches") == "samples" else 0, int(bool(st.get("recluster_hard", False))),
            int(st.get("ens_mode", 0) or 0), int(bool(st.get("skip_aggregate", False))), world,
            int(mg["rank"]) if mg else 0, int(mg["flag_base"]) if mg else 0, int(st.get("cluster", 0) or cache["cluster"]),
            spin_timeout_ms(st), int(st.get("warps_per_pair", 0) or cache["wpp"])]
    fcfg = [float(lr) if lr_dev is None else 0.0, float(st["wd"]), 0.9, 0.999, 1e-8]
    sopt = st.get("server_opt")
    sopt = None if sopt == "none" else sopt
    if sopt is not None:   # per-slot server optimizer (reference.fed_round_small documents the keys)
        from .server_opt import _KIND
        if sopt not in _KIND:
            raise ValueError(f"fed_round_small: unknown server optimizer {sopt!r}")
        icfg.append(_KIND[sopt])
        fcfg += [float(st.get("server_lr", 1.0)), float(st.get("server_momentum", 0.0)), float(st.get("server_eps", 1e-8))]
    defense = st.get("defense") or "none"
    if defense != "none":   # robust aggregation in the publish step (reference.fed_round_small documents the keys)
        from .reference import defense_params
        if len(fcfg) == 5:
            fcfg += [1.0, 0.0, 1e-8]   # server optimizer slots, unread without one
        fcfg += list(defense_params(defense, st.get("norm_bound", 5.0), st.get("stddev", 0.025)))
    prox_mu = float(st.get("fedprox_mu", 0.0) or 0.0)
    if prox_mu != 0.0:   # FedProx in every local step; the binding validates mu
        fcfg += [1.0, 0.0, 1e-8, 0.0, 0.0][len(fcfg) - 5:]   # server optimizer / defense slots, unread when off
        fcfg.append(prox_mu)
    compression = st.get("compression") or "none"
    ef_res = None
    if compression == "qsgd":   # QSGD in the publish step (reference.fed_round_small documents the keys)
        from .reference import compression_params
        q = compression_params(compression, st.get("quantize_level", 16), st.get("quantize_bucket", 512))
        fcfg += [1.0, 0.0, 1e-8, 0.0, 0.0, 0.0][len(fcfg) - 5:]   # server optimizer / defense / FedProx slots, unread when off
        fcfg += [float(q[0]), float(q[1])]
    elif compression == "eftopk":   # top-k with error feedback in the publish step; QSGD's slots stay (0, 0)
        from .reference import topk_k
        k = topk_k(st.get("topk_ratio", 0.01), theta.shape[1])
        ef_res = st.get("ef_residual")
        if ef_res is None:
            ef_res = st["ef_residual"] = torch.zeros(C, M, theta.shape[1], dtype=torch.float32, device=dev)
        fcfg += [1.0, 0.0, 1e-8, 0.0, 0.0, 0.0, 0.0, 0.0][len(fcfg) - 5:]   # server optimizer / defense / FedProx / QSGD slots
        fcfg.append(float(k))
    elif compression != "none":
        from .reference import compression_params
        compression_params(compression, 16, 512)   # raises for an unknown compression
    from .reference import aggregation_params, cclip_params, geomed_params, krum_params
    rule, beta = aggregation_params(st.get("aggregation_rule") or "mean", st.get("trim_ratio", 0.1))
    gm_iters, gm_nu = geomed_params(st.get("geomed_iters", 4), st.get("geomed_nu", 1e-6))
    krum_f, krum_m = krum_params(st.get("krum_f", 1), st.get("krum_m", 1))
    cc_tau, cc_iters = cclip_params(st.get("cclip_tau", 1.0), st.get("cclip_iters", 1))
    if rule != "mean":   # robust aggregation rule (reference.fed_round_small documents the keys)
        if mg:
            raise ValueError("a robust aggregation rule (--aggregation_rule) is single-GPU only")
        fcfg += [1.0, 0.0, 1e-8, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0][len(fcfg) - 5:]   # server optimizer ... top-k slots, unread when off
        fcfg += [float(AGG_RULE_ID[rule]), beta]
        if rule == "geometric_median":
            fcfg += [float(gm_iters), gm_nu]
        elif rule == "multi_krum":   # the geometric-median slots 16..17 are unread
            fcfg += [4.0, 1e-6, float(krum_f), float(krum_m)]
        elif rule == "centered_clip":   # the geometric-median and Multi-Krum slots 16..19 are unread
            fcfg += [4.0, 1e-6, 1.0, 1.0]
    atk, atk_a, atk_s = attack_params(st.get("attack_type") or "none", st.get("attack_clients", 0), st.get("attack_scale", 1.0),
                                      C)
    attack_mask = None
    if atk != "none" and atk_a > 0:   # simulated Byzantine clients in the publish step (reference.fed_round_small)
        if mg:
            raise ValueError("a simulated attack (--attack_type) is single-GPU only")
        attack_mask = cache.get("attack_mask")
        if attack_mask is None:
            attack_mask = cache["attack_mask"] = attack_table(st.get("attackers"), C, atk_a).to(dev, torch.uint8).contiguous()
        # server optimizer ... Multi-Krum slots, unread when off (the rule slots hold the mean and valid parameters)
        fcfg += [1.0, 0.0, 1e-8, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.1, 4.0, 1e-6, 1.0, 1.0][len(fcfg) - 5:]
        fcfg += [float(ATTACK_ID[atk]), atk_s]
    cc_center = None
    if rule == "centered_clip":   # the slots' centers, read and rewritten in place (reference.fed_round_small)
        cc_center = st.get("cclip_center")
        if cc_center is None:
            cc_center = st["cclip_center"] = torch.zeros(M, theta.shape[1], dtype=torch.float32, device=dev)
        fcfg += [0.0, 1.0][len(fcfg) - 20:]   # attack slots, unread without one
        fcfg += [cc_tau, float(cc_iters)]
    peer_metrics = []
    if mg and mg.get("metrics_ptrs") is not None:
        # every rank's LL staging area (symmetric); the kernel compacts this launch's rows into the plain metrics_out
        assert rounds <= int(mg["metrics_rounds"]), "block larger than the symmetric metrics staging area"
        peer_metrics = list(mg["metrics_ptrs"])
    info = ext.fed_round_small(
        KIND_ID[st["kind"]], int(st["din"]), int(st["hid"]), int(st["dout"]), cache["X"], cache["Y"], cache["nsamp"], W, theta,
        int(st.get("theta_stride", theta.stride(0))), st.get("opt_m"), st.get("opt_v"), st.get("opt_vmax"), st["opt_step"],
        cache["train_index"], cache["train_count"], cache["feat_mask"], cache["eval_train_model"], cache["eval_test_model"],
        ens_w, st.get("client_out"), lr_dev, metrics_out, st.get("timers"), fcfg, icfg,
        list(mg["inbox_ptrs"]) if mg else [], mg.get("error_flag") if mg else None,
        st.get("counters"), peer_metrics, [int(v) for v in st["host_io"]] if st.get("host_io") else [],
        cache["participation"], st.get("server_s0") if sopt else None, st.get("server_s1") if sopt else None,
        st.get("server_step") if sopt else None, ef_res, attack_mask, cc_center)
    if mg:
        mg["flag_base"] = int(mg["flag_base"]) + rounds
    if st.get("counters") is not None:
        st["_counter_rounds"] = st.get("_counter_rounds", 0) + rounds
    LAUNCH_COUNT["fed_round_small"] += 1
    st["round0"] = int(st["round0"]) + rounds
    st["_launch_info"] = info
    return {"metrics": metrics_out, "counts": cache["counts"]}
