"""Plain-PyTorch fp32 reference implementations of every native op.

These are (a) the CPU fallbacks and (b) the numerics oracle the GPU tests
compare the sm_90a kernels against.  Nothing here is tuned; clarity wins.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

M32 = 0xFFFFFFFF


# --------------------------------------------------------------------------- RNG
def mix32(x: int) -> int:
    """lowbias32 integer finaliser — the device RNG is the same function (csrc/common.cuh)."""
    x &= M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def batch_hash(seed: int, rnd: int, client: int, model: int, step: int) -> int:
    h = mix32((seed + 0x9E3779B9 * (rnd + 1)) & M32)
    h = mix32(h ^ ((client * 0x85EBCA6B + 0x165667B1) & M32))
    h = mix32(h ^ ((model * 0xC2B2AE35 + 0x27D4EB2F) & M32))
    h = mix32(h ^ ((step * 0x2545F491 + 1) & M32))
    return h


def hash_choice(h: int, n: int) -> int:
    """Unbiased-enough index in [0, n): high 32 bits of h·n (no modulo)."""
    return (h * n) >> 32


# --------------------------------------------------------------------------- small MLP family
def mlp_param_count(kind: str, din: int, hid: int, dout: int) -> int:
    if kind == "lr":
        return dout * din + dout
    return hid * din + hid + dout * hid + dout


def mlp_unpack(theta: torch.Tensor, kind: str, din: int, hid: int, dout: int):
    """theta [..., P] -> weight/bias views in state_dict order."""
    if kind == "lr":
        w = theta[..., : dout * din].reshape(*theta.shape[:-1], dout, din)
        b = theta[..., dout * din:]
        return w, b
    o = 0
    w1 = theta[..., o:o + hid * din].reshape(*theta.shape[:-1], hid, din); o += hid * din
    b1 = theta[..., o:o + hid]; o += hid
    w2 = theta[..., o:o + dout * hid].reshape(*theta.shape[:-1], dout, hid); o += dout * hid
    b2 = theta[..., o:o + dout]
    return w1, b1, w2, b2


def mlp_forward(theta: torch.Tensor, x: torch.Tensor, kind: str, din: int, hid: int, dout: int) -> torch.Tensor:
    """theta [P], x [B, din] -> logits-as-fed-to-CE [B, dout] (lr applies the sigmoid first)."""
    if kind == "lr":
        w, b = mlp_unpack(theta, kind, din, hid, dout)
        return torch.sigmoid(x @ w.t() + b)
    w1, b1, w2, b2 = mlp_unpack(theta, kind, din, hid, dout)
    return torch.relu(x @ w1.t() + b1) @ w2.t() + b2


def mlp_loss_grad(theta, x, y, kind, din, hid, dout):
    th = theta.detach().clone().requires_grad_(True)
    loss = F.cross_entropy(mlp_forward(th, x, kind, din, hid, dout), y.long())
    (g,) = torch.autograd.grad(loss, th)
    return loss.detach(), g


def adam_amsgrad_update(p, g, m, v, vmax, step: int, lr, wd, b1=0.9, b2=0.999, eps=1e-8):
    """torch.optim.Adam(amsgrad=True, weight_decay=wd) single-tensor semantics; in place; returns new step."""
    step += 1
    g = g + wd * p
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    torch.maximum(vmax, v, out=vmax)
    bc1 = 1 - b1 ** step
    bc2 = 1 - b2 ** step
    denom = vmax.sqrt() / math.sqrt(bc2) + eps
    p.addcdiv_(m, denom, value=-(lr / bc1))
    return step


def prox_grad(g, w, prox, r: int = 0):
    """FedProx (``--fedprox_mu``): the gradient of F(w) + μ/2‖mask ⊙ (w − a)‖², i.e. g + μ·mask ⊙ (w − a), for row r of a
    row optimizer; ``prox = (mu, anchor, anchor_rows, mask)``, a = anchor[anchor_rows[r], :P] (anchor_rows None: anchor is the
    row itself), mask a [≥ P] entry mask or None (every entry)."""
    mu, anchor, rows, mask = prox
    P = w.shape[-1]
    a = anchor if rows is None else anchor[int(rows[r])]
    d = w - a[:P]
    if mask is not None:
        d = d * mask[:P].to(d.dtype)
    return g + float(mu) * d


def mlp_eval(theta, x, y, n, kind, din, hid, dout) -> Tuple[float, float]:
    """-> (correct, loss_sum) over the first n samples."""
    if n == 0:
        return 0.0, 0.0
    logits = mlp_forward(theta, x[:n], kind, din, hid, dout)
    loss = F.cross_entropy(logits, y[:n].long(), reduction="sum")
    correct = (logits.argmax(-1) == y[:n]).sum()
    return float(correct), float(loss)


def mlp_eval_matrix(theta, X, Y, nsamp, kind, din, hid, dout):
    """theta [M,P]; X [C,S,din]; Y [C,S]; nsamp [C] -> correct [M,C], loss_sum [M,C] (fp32)."""
    M, C = theta.shape[0], X.shape[0]
    correct = torch.zeros(M, C, dtype=torch.float32, device=theta.device)
    loss = torch.zeros(M, C, dtype=torch.float32, device=theta.device)
    for m in range(M):
        for c in range(C):
            k, l = mlp_eval(theta[m], X[c], Y[c], int(nsamp[c]), kind, din, hid, dout)
            correct[m, c], loss[m, c] = k, l
    return correct, loss


def _np_view(st, nb):
    """Host-side numpy mirrors of the plan tensors (built once per `st`): scalar indexing of torch tensors costs a few
    µs per access, which dominated the per-pair sampler of the generic executor."""
    cache = st.get("_np")
    if cache is None or cache["W_id"] is not st["W"]:
        cache = st["_np"] = {"W_id": st["W"], "W": st["W"].detach().cpu().double().numpy(),
                             "nsamp": st["nsamp"].detach().cpu().numpy().astype(np.int64),
                             "nb": nb.detach().cpu().numpy().astype(np.int64),
                             "tc": st["train_count"].detach().cpu().numpy() if st.get("train_count") is not None else None}
    return cache


def _pair_plan(st, c, m, t, nb, B):
    """-> (n_cm, sampler) for (client c, model m); sampler(h1, h2) -> (sample index tensor into X[·, c])."""
    v = _np_view(st, nb)
    Wn, nsn, nbn = v["W"], v["nsamp"], v["nb"]
    mode = st.get("sample_mode", "pool")
    if mode == "index":
        cnt = int(v["tc"][m, c])
        if cnt <= 0:
            return 0.0, None
        lst = st["train_index"][m, c, :cnt].long()
        nbm = (cnt + B - 1) // B

        def sampler(h1, h2):
            b = hash_choice(h1, nbm)
            return lst[b * B:min((b + 1) * B, cnt)]
        return float(cnt), sampler
    S = st["X"].shape[2]
    wcol = Wn[: t + 1, m, c]
    nbc, nsc = nbn[: t + 1, c], nsn[: t + 1, c]
    if mode == "time":
        tot = float(wcol.sum())
        if tot <= 0:
            return 0.0, None
        n_cm = float(nbc.sum())
        cum = np.cumsum(wcol.astype(np.float32), dtype=np.float32)

        def sampler(h1, h2):
            u = np.float32(h1 >> 8) * np.float32(1.0 / 16777216.0) * np.float32(cum[-1])
            tt = min(int((cum <= u).sum()), t)
            while int(nbc[tt]) == 0 and tt > 0:
                tt -= 1
            b = hash_choice(h2, max(int(nbc[tt]), 1))
            lo, hi = b * B, min((b + 1) * B, int(nsc[tt]))
            return torch.from_numpy(np.arange(tt * S + lo, tt * S + hi, dtype=np.int64))
        return n_cm, sampler
    n_cm = float((wcol * nbc).sum())
    if n_cm <= 0:
        return 0.0, None
    pool = [(tt, b) for tt in range(t + 1) if wcol[tt] * nbc[tt] > 0 for b in range(int(nbc[tt]))]
    if st.get("n_mode", "batches") == "samples":
        n_cm = float((wcol * nsc).sum())

    def sampler(h1, h2):
        tt, b = pool[hash_choice(h1, len(pool))]
        lo, hi = b * B, min((b + 1) * B, int(nsc[tt]))
        return torch.from_numpy(np.arange(tt * S + lo, tt * S + hi, dtype=np.int64))
    return n_cm, sampler


def fed_round_small(st: Dict, rounds: int = 1) -> Dict[str, torch.Tensor]:
    """Reference semantics of the fused persistent round kernel (csrc/fed_round_small.cu).

    ``st`` keys — spec: kind,din,hid,dout; data: X [T1,C,S,din], Y [T1,C,S] int, nsamp [T1,C] int;
    batch_size; W [T,M,C] float (T ≥ t_cur+1); theta [M,P]; opt_m/opt_v/opt_vmax [C,M,P]; opt_step [C,M] int;
    hyper: lr (float or 1-elem tensor), wd, epochs, optimizer ('adam'|'sgd'), seed, round0, t_cur.
    Training-set selection (``sample_mode``):
      'pool'  — uniform over the batches of every past step t' with W[t',m,c]·nb > 0; n = Σ W·nb
                (``FedAvgEnsTrainerSoftCluster.py:72-113``); ``n_mode='samples'`` weights by Σ W·nsamp instead;
      'time'  — t' ~ W[·,m,c], then a uniform batch of t'; n = Σ_t' nb (``FedAvgEnsTrainerExp.py:55-75``);
      'index' — explicit per-(m,c) sample lists ``train_index [M,C,L]`` / ``train_count [M,C]`` (window concat,
                replication, Poisson bootstrap, client-select); batches are chunks of the list; n = list length
                (``FedAvgEnsTrainer.py:54-75``).
    Optional: ``feat_mask [M,din]`` (training inputs only, KUE), ``recluster_hard`` (IFCA per-round argmax
    re-clustering), ``eval_train_model``/``eval_test_model`` [C] int (-1 → argmax_m W[t,m,c]),
    ``ens_mode`` 0|1 (weighted hard vote)|2 (weighted soft vote) with ``ens_w [C,M]`` for the TEST metric.
    ``participation [rows, C]`` bool/uint8: in round ``rnd`` only the clients of row ``rnd % rows`` train and enter the
    cluster averages (a cluster with no participant keeps its model); evaluation and re-clustering still cover every client.
    ``server_opt`` 'sgd'|'adam'|'adagrad'|'yogi' (absent or 'none': plain FedAvg) with ``server_lr`` (1.0),
    ``server_momentum`` (0.0), ``server_eps`` (1e-8), state ``server_s0`` / ``server_s1`` [M,P] and ``server_step`` [M] int:
    every slot whose total weight is > 0 becomes avg_m, then takes one ``server_opt_slots_`` step on θ_m − avg_m; the other
    slots keep θ, state and counter (see ``server_opt.SlotServerOpt`` for which state rows each optimizer uses).
    ``defense`` 'norm_diff_clipping'|'weak_dp' (absent or 'none': off) with ``norm_bound`` (5.0) and ``stddev`` (0.025, weak_dp
    only): before the average, every trained pair's local model goes through ``robust_clip_slots_`` against the round-start θ
    with seed ``defense_seed(seed, rnd)``; the weights are unchanged.  ``compression`` 'qsgd' (absent or 'none': off) with
    ``quantize_level`` s (16) and ``quantize_bucket`` b (512): right after local training, every trained pair's local model
    goes through ``qsgd_slots_`` against the round-start θ with seed ``compress_seed(seed, rnd)`` (the client quantizes
    before it uploads), so ``client_out``, the defense and the average see the quantized model.  ``client_out [C, M, P]``:
    the local models as uploaded (quantized, undefended) of the pairs that trained in the last round are written there.
    ``compression`` 'eftopk' with ``topk_ratio`` ρ (0.01) and state ``ef_residual [C, M, P]`` (created zero when missing,
    updated in place like the optimizer moments): at the same point every trained pair's local model goes through
    ``eftopk_slots_`` against the round-start θ with k = ``topk_k(ρ, P)``; ``client_out``, the defense and the average see
    the sparsified model.
    ``aggregation_rule`` 'median'|'trimmed_mean' (absent or 'mean': the weighted average) with ``trim_ratio`` β (0.1,
    validated whatever the rule by ``aggregation_params``): after compression and the defense, every slot with a
    participant becomes ``robust_aggregate_slots_`` of its trained pairs' uploads (each counts once, the weights are
    ignored) instead of the weighted average; the server optimizer then steps on θ_m − that statistic.
    ``aggregation_rule`` 'geometric_median' with ``geomed_iters`` R (4) and ``geomed_nu`` ν (1e-6), validated whatever the
    rule by ``geomed_params``: the same, with ``geomed_aggregate_slots_`` (every entry is trainable in these MLPs).
    ``aggregation_rule`` 'multi_krum' with ``krum_f`` f (1) and ``krum_m`` m (1), validated whatever the rule by
    ``krum_params``: the same, with ``krum_aggregate_slots_``.
    ``aggregation_rule`` 'centered_clip' with ``cclip_tau`` τ (1.0) and ``cclip_iters`` L (1), validated whatever the
    rule by ``cclip_params``, and state ``cclip_center [M, P]`` (created zero when missing, updated in place like the
    optimizer moments): the same, with ``cclip_aggregate_slots_`` around the round-start θ; the server optimizer steps on
    θ_m − (θ_m + v).
    ``attack_type`` 'sign_flip'|'gaussian'|'alie'|'ipm' (absent or 'none': off) with ``attack_clients`` a (0) and
    ``attack_scale`` s (1.0), validated whatever the type by ``attack_params``, and ``attackers`` (bool/uint8 [C], absent:
    ``attacker_clients(C, a, 0)``, which must hold a clients): after compression and before ``client_out``, the defense
    and the rule, the uploads go through ``attack_slots_`` with seed ``attack_seed(seed, rnd)``.
    ``fedprox_mu`` (absent or 0: off): every local
    step of pair (c, m) feeds ``prox_grad(g, w, (mu, θ_m, None, None))`` to the client optimizer, θ_m the round-start model
    (FedProx: the local objective gains μ/2‖w − θ_m‖²; Adam adds wd·w after it).
    Mutates theta / opt state / W (if recluster) in place; returns ``metrics [rounds, C, 4]`` =
    (train_correct, train_loss_sum, test_correct, test_loss_sum) and ``counts [C, 2]`` = (n_train, n_test).
    """
    kind, din, hid, dout = st["kind"], st["din"], st["hid"], st["dout"]
    X, Y, nsamp, W, theta = st["X"], st["Y"], st["nsamp"], st["W"], st["theta"]
    B, E, t = int(st["batch_size"]), int(st["epochs"]), int(st["t_cur"])
    T1, C, S = X.shape[0], X.shape[1], X.shape[2]
    M, P = theta.shape
    wd = float(st["wd"])
    use_adam = st.get("optimizer", "adam") != "sgd"
    seed, round0 = int(st["seed"]), int(st["round0"])
    nb = (nsamp.to(torch.int64) + B - 1) // B  # [T1, C] batches per (t, c)
    metrics = torch.zeros(rounds, C, 4, dtype=torch.float32)
    feat_mask = st.get("feat_mask")
    ens_mode = int(st.get("ens_mode", 0) or 0)
    Xflat = X.reshape(T1, C, S, -1)
    part = st.get("participation")
    if part is not None:
        part = torch.as_tensor(part).to("cpu", torch.bool)
    sopt = st.get("server_opt")
    if sopt == "none":
        sopt = None
    defense = st.get("defense") or "none"
    def_bound, def_std = defense_params(defense, st.get("norm_bound", 5.0), st.get("stddev", 0.025))
    prox_mu = prox_mu_param(st.get("fedprox_mu", 0.0))
    q_level, q_bucket = compression_params(st.get("compression") or "none", st.get("quantize_level", 16),
                                           st.get("quantize_bucket", 512))
    ef_ratio = topk_ratio_param(st.get("topk_ratio", 0.01))
    ef_k = topk_k(ef_ratio, P) if (st.get("compression") or "none") == "eftopk" else 0
    if ef_k and st.get("ef_residual") is None:
        st["ef_residual"] = torch.zeros(C, M, P, dtype=torch.float32)
    agg_rule, trim_ratio = aggregation_params(st.get("aggregation_rule") or "mean", st.get("trim_ratio", 0.1))
    gm_iters, gm_nu = geomed_params(st.get("geomed_iters", 4), st.get("geomed_nu", 1e-6))
    krum_f, krum_m = krum_params(st.get("krum_f", 1), st.get("krum_m", 1))
    cc_tau, cc_iters = cclip_params(st.get("cclip_tau", 1.0), st.get("cclip_iters", 1))
    if agg_rule == "centered_clip" and st.get("cclip_center") is None:
        st["cclip_center"] = torch.zeros(M, P, dtype=torch.float32)
    atk_type, atk_a, atk_scale = attack_params(st.get("attack_type") or "none", st.get("attack_clients", 0),
                                               st.get("attack_scale", 1.0), C)
    attackers = attack_table(st.get("attackers"), C, atk_a)
    atk_on = atk_type != "none" and atk_a > 0
    client_out = st.get("client_out")
    for r in range(rounds):
        rnd = round0 + r
        prow = part[rnd % part.shape[0]] if part is not None else None
        cur_lr = float(st["lr"])
        Wt = W[t]
        if st.get("sample_mode", "pool") == "index":
            active = (st["train_count"] > 0).any(dim=1)
        else:
            active = (Wt != 0).any(dim=1)  # [M]
        acc_w = torch.zeros(M, dtype=torch.float64)
        locals_: Dict[Tuple[int, int], Tuple[torch.Tensor, float]] = {}
        for c in range(C):
            if prow is not None and not bool(prow[c]):
                continue
            Xc = Xflat[:, c].reshape(T1 * S, -1)
            Yc = Y[:, c].reshape(T1 * S)
            for m in range(M):
                if not bool(active[m]):
                    continue
                n_cm, sampler = _pair_plan(st, c, m, t, nb, B)
                if n_cm <= 0:
                    continue
                p = theta[m].clone()
                for step in range(E):
                    h1 = batch_hash(seed, rnd, c, m, step)
                    idx = sampler(h1, mix32(h1 ^ 0x68E31DA4))
                    xb, yb = Xc[idx], Yc[idx]
                    if feat_mask is not None:
                        xb = xb * feat_mask[m]
                    _, g = mlp_loss_grad(p, xb, yb, kind, din, hid, dout)
                    if prox_mu > 0:
                        g = prox_grad(g, p, (prox_mu, theta[m], None, None))
                    if use_adam:
                        st["opt_step"][c, m] = adam_amsgrad_update(
                            p, g, st["opt_m"][c, m], st["opt_v"][c, m], st["opt_vmax"][c, m],
                            int(st["opt_step"][c, m]), cur_lr, wd)
                    else:
                        p.add_(g, alpha=-cur_lr)
                locals_[(c, m)] = (p, n_cm)
                acc_w[m] += n_cm
        if q_level and locals_:   # QSGD: each client quantizes its upload against the round-start θ_m
            up = torch.zeros(C, M, P, dtype=torch.float32)
            trained = torch.zeros(C, M)
            for (c, m), (p, _) in locals_.items():
                up[c, m], trained[c, m] = p, 1.0
            qsgd_slots_(up, theta, trained, q_level, q_bucket, None, compress_seed(seed, rnd))
            locals_ = {(c, m): (up[c, m], n_cm) for (c, m), (_, n_cm) in locals_.items()}
        if ef_k and locals_:   # top-k with error feedback: each client sparsifies its upload against the round-start θ_m
            up = torch.zeros(C, M, P, dtype=torch.float32)
            trained = torch.zeros(C, M)
            for (c, m), (p, _) in locals_.items():
                up[c, m], trained[c, m] = p, 1.0
            eftopk_slots_(up, theta, st["ef_residual"], trained, ef_k, None)
            locals_ = {(c, m): (up[c, m], n_cm) for (c, m), (_, n_cm) in locals_.items()}
        if atk_on and locals_:   # the Byzantine clients replace their uploads as they leave (after compression)
            up = torch.zeros(C, M, P, dtype=torch.float32)
            trained = torch.zeros(C, M)
            for (c, m), (p, _) in locals_.items():
                up[c, m], trained[c, m] = p, 1.0
            attack_slots_(up, theta, trained, attackers, atk_type, atk_scale, None, attack_seed(seed, rnd))
            locals_ = {(c, m): (up[c, m], n_cm) for (c, m), (_, n_cm) in locals_.items()}
        if client_out is not None and r == rounds - 1:
            for (c, m), (p, _) in locals_.items():
                client_out[c, m] = p
        if defense != "none" and locals_:
            up = torch.zeros(C, M, P, dtype=torch.float32)
            for (c, m), (p, _) in locals_.items():
                up[c, m] = p
            trained = torch.zeros(C, M)
            for (c, m) in locals_:
                trained[c, m] = 1.0
            robust_clip_slots_(up, theta, trained, def_bound, None, def_std, defense_seed(seed, rnd))
            locals_ = {(c, m): (up[c, m], n_cm) for (c, m), (_, n_cm) in locals_.items()}
        avg = theta.clone() if sopt is not None else theta
        if agg_rule != "mean" and locals_:   # robust rule: every participant counts once, the weights are ignored
            up = torch.zeros(C, M, P, dtype=torch.float32)
            trained = torch.zeros(C, M)
            for (c, m), (p, _) in locals_.items():
                up[c, m], trained[c, m] = p, 1.0
            if agg_rule == "geometric_median":
                geomed_aggregate_slots_(avg, up, trained, gm_iters, gm_nu)
            elif agg_rule == "multi_krum":
                krum_aggregate_slots_(avg, up, trained, krum_f, krum_m)
            elif agg_rule == "centered_clip":
                cclip_aggregate_slots_(avg, up, trained, st["cclip_center"], cc_tau, cc_iters)
            else:
                robust_aggregate_slots_(avg, up, trained, agg_rule, trim_ratio)
        for m in range(M):
            if acc_w[m] <= 0 or agg_rule != "mean":
                continue
            tot = np.float32(acc_w[m])
            out = torch.zeros(P, dtype=torch.float32)
            for c in range(C):
                if (c, m) in locals_:
                    p, n_cm = locals_[(c, m)]
                    out += p * (np.float32(n_cm) / tot)
            avg[m] = out
        if sopt is not None:
            server_opt_slots_(theta, avg, acc_w > 0, sopt, st.get("server_s0"), st.get("server_s1"), st["server_step"],
                              float(st.get("server_lr", 1.0)), float(st.get("server_momentum", 0.0)),
                              float(st.get("server_eps", 1e-8)))
        if st.get("recluster_hard", False):
            corr, _ = mlp_eval_matrix(theta, Xflat[t], Y[t], nsamp[t], kind, din, hid, dout)
            accm = corr / nsamp[t].clamp(min=1).float()
            best = accm.argmax(dim=0)  # first max == np.argmax tie-break
            W[t].zero_()
            W[t][best, torch.arange(C)] = 1.0
            st.pop("_np", None)   # the numpy mirror of W is stale
        pick = W[t].argmax(dim=0)
        etr, ete = st.get("eval_train_model"), st.get("eval_test_model")
        for c in range(C):
            mtr = int(etr[c]) if etr is not None and int(etr[c]) >= 0 else int(pick[c])
            mte = int(ete[c]) if ete is not None and int(ete[c]) >= 0 else int(pick[c])
            k, l = mlp_eval(theta[mtr], Xflat[t, c], Y[t, c], int(nsamp[t, c]), kind, din, hid, dout)
            metrics[r, c, 0], metrics[r, c, 1] = k, l
            if t + 1 < T1:
                n1 = int(nsamp[t + 1, c])
                if ens_mode == 0:
                    k, l = mlp_eval(theta[mte], Xflat[t + 1, c], Y[t + 1, c], n1, kind, din, hid, dout)
                elif n1 > 0:
                    tally = torch.zeros(n1, dout, dtype=torch.float32)
                    for m in range(M):
                        w = float(st["ens_w"][c, m])
                        if w <= 0:
                            continue
                        lg = mlp_forward(theta[m], Xflat[t + 1, c, :n1], kind, din, hid, dout)
                        if ens_mode == 1:
                            tally[torch.arange(n1), lg.argmax(-1)] += np.float32(w)
                        else:
                            tally += np.float32(w) * F.softmax(lg, dim=1)
                    k, l = float((tally.argmax(-1) == Y[t + 1, c, :n1]).sum()), 0.0
                else:
                    k, l = 0.0, 0.0
                metrics[r, c, 2], metrics[r, c, 3] = k, l
    counts = torch.stack([nsamp[t], nsamp[t + 1] if t + 1 < T1 else torch.zeros_like(nsamp[t])], dim=1).float()
    st["round0"] = round0 + rounds
    return {"metrics": metrics, "counts": counts}


# --------------------------------------------------------------------------- K1 / K8 / K10 / K11 / K12
def cluster_aggregate_(theta: torch.Tensor, client_params: torch.Tensor, n: torch.Tensor) -> torch.Tensor:
    """theta [M,P] <- per-model weighted mean of client_params [C,M,P] with weights n [C,M]
    (models whose total weight is 0 are left untouched).  Returns totals [M]."""
    tot = n.double().sum(0)  # [M]
    for m in range(theta.shape[0]):
        if tot[m] > 0:
            w = (n[:, m].double() / tot[m]).float()
            theta[m] = (client_params[:, m, :] * w[:, None]).sum(0)
    return tot.float()


def weighted_average(rows: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
    """rows [n,P], weights [n] -> Σ w_i/Σw · row_i  (plain FedAvg, K1)."""
    w = (weights.double() / weights.double().sum()).to(rows.dtype)
    return (rows * w[:, None]).sum(0)


def _mix32_np(x):
    import numpy as np
    x = x.astype(np.uint32)
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x7FEB352D)
    x ^= x >> np.uint32(15)
    x *= np.uint32(0x846CA68B)
    x ^= x >> np.uint32(16)
    return x


def gauss_hash(seed: int, R: int, P: int) -> torch.Tensor:
    """[R, P] standard-normal noise: Box–Muller on lowbias32 hashes of (seed, row, element) — bit-compatible inputs
    with ``gauss_hash`` in csrc/common.cuh (P < 2³²)."""
    return gauss_hash_rows(seed, np.arange(R), P)


def gauss_hash_rows(seed: int, rows, P: int) -> torch.Tensor:
    """``gauss_hash`` noise of the listed row ids only: ``[len(rows), P]``."""
    with np.errstate(over="ignore"):
        i = np.arange(P, dtype=np.uint32)[None, :]
        r = np.asarray(rows, dtype=np.uint32).reshape(-1, 1)
        base = _mix32_np(np.uint32(seed & M32) ^ _mix32_np(r * np.uint32(0x9E3779B9) + np.uint32(0x7F4A7C15)))
        h1 = _mix32_np(base ^ (i * np.uint32(2) + np.uint32(1)))
        h2 = _mix32_np(base ^ (i * np.uint32(2) + np.uint32(2)) ^ np.uint32(0x68E31DA4))
    u1 = ((h1 >> np.uint32(8)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (h2 >> np.uint32(8)).astype(np.float64) / 16777216.0
    return torch.from_numpy((np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)).astype(np.float32))


def robust_clip_(rows: torch.Tensor, global_row: torch.Tensor, bound: float, weight_mask=None, stddev: float = 0.0,
                 seed: int = 0) -> torch.Tensor:
    """rows[i] <- global + (rows[i]-global)/max(1, ‖diff‖/bound) (+ stddev·N(0,1)); mask=False entries pass through (K10)."""
    diff = rows - global_row
    d = diff if weight_mask is None else diff * weight_mask
    norm = d.norm(dim=1, keepdim=True)
    scale = 1.0 / torch.clamp(norm / bound, min=1.0)
    new = global_row + diff * scale
    if stddev:
        new = new + stddev * gauss_hash(seed, rows.shape[0], rows.shape[1]).to(rows.device)
    if weight_mask is not None:
        new = torch.where(weight_mask.bool(), new, rows)
    rows.copy_(new)
    return norm.squeeze(1)


DEFENSES = ("none", "norm_diff_clipping", "weak_dp")


def defense_params(defense: str, norm_bound: float, stddev: float) -> Tuple[float, float]:
    """Validated ``(norm_bound, noise stddev)`` of a robust-aggregation defense (``--defense_type`` / ``--norm_bound`` /
    ``--stddev``); the stddev is 0 unless ``defense`` is ``weak_dp``.  Raises ``ValueError`` for an unknown defense, a
    bound that is not finite or ≤ 0, or a negative stddev."""
    if defense not in DEFENSES:
        raise ValueError(f"defense_type must be one of {', '.join(DEFENSES)} (got {defense!r})")
    bound, std = float(norm_bound), float(stddev)
    if not math.isfinite(bound) or bound <= 0.0:
        raise ValueError(f"norm_bound must be finite and > 0 (got {norm_bound!r})")
    if not math.isfinite(std) or std < 0.0:
        raise ValueError(f"stddev must be finite and >= 0 (got {stddev!r})")
    return bound, (std if defense == "weak_dp" else 0.0)


def prox_mu_param(mu) -> float:
    """Validated FedProx coefficient (``--fedprox_mu``): a finite float ≥ 0, else ``ValueError``."""
    mu = float(mu)
    if not math.isfinite(mu) or mu < 0:
        raise ValueError(f"fedprox_mu must be finite and >= 0 (got {mu})")
    return mu


def defense_seed(seed: int, rnd: int) -> int:
    """``gauss_hash`` seed of the weak-DP noise in round ``rnd`` of a time step whose engine seed is ``seed`` (the
    ``defense_seed`` of csrc/common.cuh): a function of (seed, round) only, so resumed runs, multi-round launches and
    CUDA-graph replays draw the same noise."""
    return mix32((seed & M32) ^ mix32((rnd * 0xC2B2AE35 + 0x2545F491) & M32))


def robust_clip_slots_(rows: torch.Tensor, theta: torch.Tensor, n=None, bound: float = 5.0, weight_mask=None,
                       stddev: float = 0.0, seed: int = 0) -> torch.Tensor:
    """K10 over an upload arena ``rows [C, M, P]``, in place: row (c, m) with ``n[c, m] > 0`` (every row when ``n`` is None)
    becomes θ_m + s·(row − θ_m) with s = 1 / max(1, ‖mask·(row − θ_m)‖ / bound) and θ_m = ``theta[m, :P]``, plus
    ``stddev · gauss_hash(seed, c·M + m, e)`` on every entry e.  Entries with ``weight_mask`` False pass through; a row with
    s == 1 and no noise is left bit-identical.  Returns the norms ``[C, M]`` (0 for skipped rows)."""
    C, M, P = rows.shape
    th = theta[:, :P].to(rows.device)
    sel = torch.ones(C, M, dtype=torch.bool) if n is None else (n.detach().cpu().reshape(C, M) > 0)
    wm = None if weight_mask is None else weight_mask[:P].to(rows.device).bool()
    norms = torch.zeros(C, M, dtype=torch.float32, device=rows.device)
    for c, m in sel.nonzero().tolist():
        row = rows[c, m]
        diff = row - th[m]
        nrm = (diff if wm is None else diff * wm).norm()
        norms[c, m] = nrm
        scale = 1.0 / torch.clamp(nrm / bound, min=1.0)
        if bool(scale == 1.0) and not stddev:
            continue
        new = th[m] + diff * scale
        if stddev:
            new = new + stddev * gauss_hash_rows(seed, [c * M + m], P)[0].to(rows.device)
        if wm is not None:
            new = torch.where(wm, new, row)
        row.copy_(new)
    return norms


COMPRESSIONS = ("none", "qsgd", "eftopk")


def _int_param(name: str, v) -> int:
    if isinstance(v, bool):
        raise ValueError(f"{name} must be an integer (got {v!r})")
    try:
        f = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be an integer (got {v!r})") from None
    if not math.isfinite(f) or f != int(f):
        raise ValueError(f"{name} must be an integer (got {v!r})")
    return int(f)


def compression_params(compression: str, quantize_level, quantize_bucket) -> Tuple[int, int]:
    """Validated ``(level s, bucket b)`` of the upload compression (``--compression`` / ``--quantize_level`` /
    ``--quantize_bucket``); ``(0, 0)`` for ``none`` and ``eftopk`` (QSGD off).  Raises ``ValueError`` for an unknown compression, a level that is not
    an integer in [1, 65535], or a bucket that is not an integer ≥ 1 (whatever the compression)."""
    if compression not in COMPRESSIONS:
        raise ValueError(f"compression must be one of {', '.join(COMPRESSIONS)} (got {compression!r})")
    s = _int_param("quantize_level", quantize_level)
    b = _int_param("quantize_bucket", quantize_bucket)
    if not 1 <= s <= 65535:
        raise ValueError(f"quantize_level must be in [1, 65535] (got {quantize_level!r})")
    if b < 1:
        raise ValueError(f"quantize_bucket must be >= 1 (got {quantize_bucket!r})")
    return (s, b) if compression == "qsgd" else (0, 0)


def compress_seed(seed: int, rnd: int) -> int:
    """``uniform_hash`` seed of the QSGD draws in round ``rnd`` of a time step whose engine seed is ``seed`` (the
    ``compress_seed`` of csrc/common.cuh): a function of (seed, round) only, with constants that differ from
    ``defense_seed`` so that quantization draws and weak-DP noise are independent."""
    return mix32((seed & M32) ^ mix32((rnd * 0x27D4EB2F + 0x165667B1) & M32))


def uniform_hash(seed: int, rows, P: int) -> torch.Tensor:
    """``[len(rows), P]`` float32 U[0, 1) draws of (seed, row, element): (h >> 8)·2⁻²⁴ with h the first lowbias32 hash of
    ``gauss_hash`` — bit-compatible with ``uniform_hash`` in csrc/common.cuh (P < 2³²)."""
    with np.errstate(over="ignore"):
        i = np.arange(P, dtype=np.uint32)[None, :]
        r = np.asarray(rows, dtype=np.uint32).reshape(-1, 1)
        base = _mix32_np(np.uint32(seed & M32) ^ _mix32_np(r * np.uint32(0x9E3779B9) + np.uint32(0x7F4A7C15)))
        h1 = _mix32_np(base ^ (i * np.uint32(2) + np.uint32(1)))
    return torch.from_numpy((h1 >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0))


def qsgd_slots_(rows: torch.Tensor, theta: torch.Tensor, n=None, level: int = 16, bucket: int = 512, weight_mask=None,
                seed: int = 0) -> torch.Tensor:
    """QSGD (K17) over an upload arena ``rows [C, M, P]``, in place.  Row (c, m) with ``n[c, m] > 0`` (every row when ``n``
    is None) is quantized against θ_m = ``theta[m, :P]``:

    * d = row − θ_m; entries with ``weight_mask`` False pass through and are not used below;
    * buckets are the flat ranges [k·b, (k+1)·b); σ_k = max |d_e| over the bucket's trainable entries (a max, so GPU and
      CPU agree bit for bit); a bucket with σ_k == 0 is left unchanged;
    * a = (|d_e| / σ_k)·s, q = floor(a) + (u < a − floor(a)) with u = ``uniform_hash(seed, c·M + m, e)``;
    * row_e = θ_e + copysign(σ_k·(q / s), d_e), every operation rounded in fp32.

    E[row] is the raw upload; with s = 1 every update is ternary.  Returns ``rows``."""
    C, M, P = rows.shape
    s, b = compression_params("qsgd", level, bucket)
    if C * M == 0 or P == 0:
        return rows
    b = min(b, P)
    nb = (P + b - 1) // b
    th = theta[:, :P].to(rows.device)
    sel = torch.ones(C, M, dtype=torch.bool) if n is None else (n.detach().cpu().reshape(C, M) > 0)
    wm = None if weight_mask is None else weight_mask[:P].to(rows.device).bool()
    sf = torch.tensor(float(s), dtype=torch.float32, device=rows.device)
    for c, m in sel.nonzero().tolist():
        row = rows[c, m]
        d = row - th[m]
        ad = d.abs()
        if wm is not None:
            ad = torch.where(wm, ad, torch.zeros_like(ad))
        sig = F.pad(ad, (0, nb * b - P)).view(nb, b).amax(1).repeat_interleave(b)[:P]
        a = (ad / sig) * sf
        lvl = torch.floor(a)
        u = uniform_hash(seed, [c * M + m], P)[0].to(rows.device)
        q = torch.where(u < a - lvl, lvl + 1.0, lvl)
        new = th[m] + torch.copysign(sig * (q / sf), d)
        keep = sig == 0
        if wm is not None:
            keep = keep | ~wm
        row.copy_(torch.where(keep, row, new))
    return rows


def qsgd_upload_bits(P_train: int, P_other: int, level: int, bucket: int, weight_mask=None) -> int:
    """Fixed-length code size in bits of one QSGD upload: 32 bits per bucket holding at least one trainable entry, plus
    1 + ⌈log₂(s+1)⌉ bits (sign and level) per trainable entry, plus 32 bits per non-trainable entry (sent raw).  The
    buckets are counted from ``weight_mask`` (bool [P_train + P_other]) when given; without it the trainable entries are
    taken to be contiguous, so ⌈P_train / b⌉ buckets hold them."""
    s, b = compression_params("qsgd", level, bucket)
    P_train, P_other = int(P_train), int(P_other)
    if weight_mask is not None:
        wm = torch.as_tensor(weight_mask)[: P_train + P_other].bool().cpu()
        if int(wm.sum()) != P_train:
            raise ValueError("weight_mask must hold exactly P_train trainable entries")
        P = P_train + P_other
        nb = (P + b - 1) // b
        buckets = int((F.pad(wm.to(torch.uint8), (0, nb * b - P)).view(nb, b).amax(1) > 0).sum()) if P else 0
    else:
        buckets = (P_train + b - 1) // b
    return 32 * buckets + (1 + int(s).bit_length()) * P_train + 32 * P_other


def topk_ratio_param(rho) -> float:
    """Validated ``--topk_ratio`` ρ (fraction of the trainable entries an ``eftopk`` upload keeps): a finite number with
    0 < ρ ≤ 1, checked whatever the compression.  Raises ``ValueError`` otherwise."""
    if isinstance(rho, bool):
        raise ValueError(f"topk_ratio must be a number in (0, 1] (got {rho!r})")
    try:
        f = float(rho)
    except (TypeError, ValueError):
        raise ValueError(f"topk_ratio must be a number in (0, 1] (got {rho!r})") from None
    if not (math.isfinite(f) and 0.0 < f <= 1.0):
        raise ValueError(f"topk_ratio must be a number in (0, 1] (got {rho!r})")
    return f


def topk_k(rho, n_train: int) -> int:
    """Entries kept per ``eftopk`` upload: max(1, min(n_train, ⌊ρ·n_train + 0.5⌋)) over ``n_train`` trainable entries
    (round half up in float64; ⌈ρ·n⌉ would give 4 for ρ = 0.1, n = 30)."""
    f = topk_ratio_param(rho)
    n_train = int(n_train)
    return max(1, min(n_train, int(math.floor(f * n_train + 0.5))))


def eftopk_slots_(rows: torch.Tensor, theta: torch.Tensor, residual: torch.Tensor, n=None, k: int = 1,
                  weight_mask=None) -> torch.Tensor:
    """Top-k sparsification with error feedback (K18) over an upload arena ``rows [C, M, P]`` and its residual
    ``residual [C, M, P]``, both in place.  Row (c, m) with ``n[c, m] > 0`` (every row when ``n`` is None), with
    θ_m = ``theta[m, :P]``, x the row and e its residual:

    * v = (x − θ_m) + e over the trainable entries (``weight_mask`` True), each operation rounded in fp32;
    * key = bit pattern of |v| as uint32; the k entries with the largest keys are selected, ties going to the lower flat
      index (a total order, so GPU and CPU agree bit for bit);
    * a selected entry uploads x + e (x itself when e == 0) and its residual becomes 0;
    * an unselected trainable entry uploads θ_e and its residual becomes v;
    * non-trainable entries pass through and keep their residual.

    Rows with n ≤ 0 keep both their upload and their residual.  With k ≥ the trainable count every entry is selected, so
    a zero residual stays zero and the uploads are unchanged.  Returns ``rows``."""
    C, M, P = rows.shape
    k = int(k)
    if k < 1:
        raise ValueError(f"eftopk: k must be >= 1 (got {k})")
    if tuple(residual.shape) != (C, M, P):
        raise ValueError("eftopk: residual must have the shape of rows")
    if C * M == 0 or P == 0:
        return rows
    th = theta[:, :P].to(rows.device)
    sel = torch.ones(C, M, dtype=torch.bool) if n is None else (n.detach().cpu().reshape(C, M) > 0)
    wm = torch.ones(P, dtype=torch.bool, device=rows.device) if weight_mask is None else \
        weight_mask[:P].to(rows.device).bool()
    cand = wm.nonzero().flatten()
    kk = min(k, int(cand.numel()))
    for c, m in sel.nonzero().tolist():
        x, e = rows[c, m], residual[c, m]
        v = (x - th[m]) + e
        key = v.view(torch.int32).to(torch.int64) & 0x7FFFFFFF
        order = torch.sort(key[cand], descending=True, stable=True).indices[:kk]
        chosen = torch.zeros(P, dtype=torch.bool, device=rows.device)
        chosen[cand[order]] = True
        up = torch.where(e == 0, x, x + e)
        new_x = torch.where(chosen, up, torch.where(wm, th[m], x))
        new_e = torch.where(chosen, torch.zeros_like(e), torch.where(wm, v, e))
        x.copy_(new_x)
        e.copy_(new_e)
    return rows


def topk_upload_bits(P_train: int, P_other: int, k: int) -> int:
    """Size in bits of one ``eftopk`` upload: a 32-bit value and a ⌈log₂ P⌉-bit index (bit_length(P − 1)) per kept entry,
    plus 32 bits per non-trainable entry (sent raw), with P = P_train + P_other."""
    P_train, P_other, k = int(P_train), int(P_other), int(k)
    P = P_train + P_other
    return k * (32 + max(P - 1, 0).bit_length()) + 32 * P_other


# Multi-Krum has one name: ``multi_krum`` with ``krum_m`` = 1 is plain Krum, and a bare ``krum`` is an unknown rule.
AGGREGATION_RULES = ("mean", "median", "trimmed_mean", "geometric_median", "multi_krum", "centered_clip")


def aggregation_params(rule, trim_ratio) -> Tuple[str, float]:
    """Validated ``(--aggregation_rule, --trim_ratio)``.  The rule is one of ``mean`` (weighted FedAvg), ``median``,
    ``trimmed_mean``, ``geometric_median``, ``multi_krum`` or ``centered_clip``; β is checked whatever the rule and must
    be a finite number with 0 ≤ β < 0.5.  Raises ``ValueError``."""
    rule = "mean" if rule is None else rule
    if rule not in AGGREGATION_RULES:
        raise ValueError(f"aggregation_rule must be one of {', '.join(AGGREGATION_RULES)} (got {rule!r})")
    msg = f"trim_ratio must be a number in [0, 0.5) (got {trim_ratio!r})"
    if isinstance(trim_ratio, bool):
        raise ValueError(msg)
    try:
        b = float(trim_ratio)
    except (TypeError, ValueError):
        raise ValueError(msg) from None
    if not (math.isfinite(b) and 0.0 <= b < 0.5):
        raise ValueError(msg)
    return rule, b


def trim_count(beta, n: int) -> int:
    """Values ``trimmed_mean`` drops at EACH end of a column of ``n`` uploads: ⌊fl32(fl32(β)·n)⌋, one fp32 rounding of the
    product (``np.float32(β) * np.float32(n)``), so CPU and GPU agree.  β < 0.5 keeps at least one value."""
    return int(np.floor(np.float32(beta) * np.float32(int(n))))


_QNAN32 = np.uint32(0x7FC00000).view(np.float32).item()   # the NaN a column containing a NaN yields (GPU: same bits)


def robust_aggregate_slots_(theta: torch.Tensor, uploads: torch.Tensor, n: torch.Tensor, rule: str = "median",
                            trim_ratio: float = 0.1) -> torch.Tensor:
    """Coordinate-wise robust aggregation (K19), in place: for every slot m, the participants are the rows c with
    ``n[c, m] > 0`` (n of them; the weights are otherwise ignored: each participant counts once, so a client cannot buy
    influence by reporting a large sample count).  For each entry e of ``theta[m, :P]`` (``theta`` may be a padded bank;
    every entry, BatchNorm statistics included):

    * the rank of upload i is #{j : a_j < a_i} + #{j < i : a_j == a_i}, compared as floats (−0 and +0 tie);
    * ``median`` keeps ranks b … n−1−b with b = ⌊(n − 1)/2⌋, ``trimmed_mean`` with b = ``trim_count(β, n)``;
    * the value is the fp32 sum of the kept values in ascending rank order, starting from the smallest kept one, then one
      round-to-nearest division by (n − 2b); a column that holds a NaN yields NaN.

    The result depends only on the multiset of uploads (any client permutation gives the same bits).  Slots with n = 0
    keep θ_m.  Returns the per-slot participant counts ``[M]`` (float32)."""
    rule, beta = aggregation_params(rule, trim_ratio)
    if rule not in ("median", "trimmed_mean"):
        raise ValueError("robust_aggregate_slots_: rule must be median or trimmed_mean (the mean is cluster_aggregate_, the "
                         "geometric median geomed_aggregate_slots_)")
    C, M, P = uploads.shape
    part = n.detach().reshape(C, M).to(uploads.device) > 0
    counts = part.sum(0).to(torch.float32)
    chunk = 1 << 20
    for m in range(M):
        idx = part[:, m].nonzero().flatten()
        k = int(idx.numel())
        if k == 0:
            continue
        b = (k - 1) // 2 if rule == "median" else trim_count(beta, k)
        div = torch.tensor(float(k - 2 * b), dtype=torch.float32, device=uploads.device)
        for e0 in range(0, P, chunk):
            vals = uploads[idx, m, e0:e0 + chunk].to(torch.float32)
            # stable ascending sort on +0-canonicalised keys: equal values (−0 and +0 included) stay in client order
            order = torch.sort(vals + 0.0, dim=0, stable=True).indices
            srt = torch.gather(vals, 0, order)
            acc = srt[b].clone()
            for j in range(b + 1, k - b):
                acc = acc + srt[j]
            out = acc / div
            out = torch.where(torch.isnan(vals).any(0), torch.full_like(out, _QNAN32), out)
            theta[m, e0:e0 + out.shape[0]] = out.to(theta.device)
    return counts.to(theta.device)


GEOMED_MAX_ITERS = 100


def geomed_params(iters, nu) -> Tuple[int, float]:
    """Validated ``(--geomed_iters, --geomed_nu)``, checked whatever the rule: R an int with 1 ≤ R ≤ 100 (a bool is not
    an int here), ν a finite number > 0.  Raises ``ValueError``."""
    if isinstance(iters, bool) or not isinstance(iters, (int, np.integer)) or not 1 <= int(iters) <= GEOMED_MAX_ITERS:
        raise ValueError(f"geomed_iters must be an int in [1, {GEOMED_MAX_ITERS}] (got {iters!r})")
    msg = f"geomed_nu must be a finite number > 0 (got {nu!r})"
    if isinstance(nu, bool):
        raise ValueError(msg)
    try:
        v = float(nu)
    except (TypeError, ValueError):
        raise ValueError(msg) from None
    if not (math.isfinite(v) and v > 0.0):
        raise ValueError(msg)
    return int(iters), v


def geomed_aggregate_slots_(theta: torch.Tensor, uploads: torch.Tensor, n: torch.Tensor, iters: int = 4, nu: float = 1e-6,
                            mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Geometric median (K20, RFA's smoothed Weiszfeld iteration), in place.  For every slot m the participants x_1…x_n are
    the rows c with ``n[c, m] > 0`` in ascending c, each counted once (the weights are ignored, as in
    ``robust_aggregate_slots_``); ``theta`` may be a padded bank.

    * Start: v⁰ = the coordinate-wise median (``robust_aggregate_slots_(…, "median")``).  With n ≤ 2 that is the result.
    * Iteration t = 1…R (R = ``iters``):
      d_i² = Σ_e mask_e · (double) fl32(x_ie − v_e)², the fp32 difference squared and summed in float64 (``mask``: the
      trainable entries, None = all, so BatchNorm statistics stay out of the distance);
      w_i = fl32(1 / max(ν, √d_i²)) computed in float64 and rounded once (d_i = +∞ gives w_i = 0: the row is left out);
      W = the fp32 sum of the w_i in client order;
      v_e = fl32(Σ_i fl32(w_i · x_ie)) summed in client order from 0 over the rows with w_i ≠ 0, then one round-to-nearest
      division by W, for every entry (BatchNorm statistics included).
    * W = 0 keeps the current v (and every later iteration would too).  A NaN distance makes the slot NaN (0x7FC00000)
      in every entry.

    The float64 distance sums depend on the reduction order, so the GPU matches this to a tolerance; given identical
    weights the update is bit-exact.  Slots with n = 0 keep θ_m.  Returns the per-slot participant counts ``[M]``."""
    R, nu = geomed_params(iters, nu)
    counts = robust_aggregate_slots_(theta, uploads, n, "median")
    C, M, P = uploads.shape
    dev = uploads.device
    part = n.detach().reshape(C, M).to(dev) > 0
    keep = None if mask is None else mask.reshape(-1)[:P].to(dev, torch.bool)
    chunk = 1 << 20
    for m in range(M):
        idx = part[:, m].nonzero().flatten().tolist()
        k = len(idx)
        if k <= 2:
            continue
        v = theta[m, :P].to(dev, torch.float32).clone()
        for _ in range(R):
            d2 = torch.zeros(k, dtype=torch.float64, device=dev)
            for e0 in range(0, P, chunk):
                diff = (uploads[idx, m, e0:e0 + chunk].to(torch.float32) - v[e0:e0 + chunk]).double()
                sq = diff * diff
                if keep is not None:
                    sq = torch.where(keep[e0:e0 + chunk], sq, torch.zeros((), dtype=torch.float64, device=dev))
                d2 += sq.sum(1)
            if bool(torch.isnan(d2).any()):
                v.fill_(_QNAN32)
                break
            w = (1.0 / torch.clamp(torch.sqrt(d2), min=nu)).to(torch.float32)
            W = np.float32(0.0)
            for wi in w.tolist():
                W = np.float32(W + np.float32(wi))
            if W == 0:
                break
            rows = [i for i in range(k) if float(w[i]) != 0.0]
            div = torch.tensor(float(W), dtype=torch.float32, device=dev)
            new = torch.empty_like(v)
            for e0 in range(0, P, chunk):
                acc = torch.zeros(min(chunk, P - e0), dtype=torch.float32, device=dev)
                for i in rows:
                    acc = acc + w[i] * uploads[idx[i], m, e0:e0 + chunk].to(torch.float32)
                new[e0:e0 + chunk] = acc / div
            v = new
        theta[m, :P] = v.to(theta.device)
    return counts


KRUM_MAX = 65535


def krum_params(f, m) -> Tuple[int, int]:
    """Validated ``(--krum_f, --krum_m)``, checked whatever the rule: f an int with 0 ≤ f ≤ 65535 (the Byzantine uploads a
    slot is assumed to hold), m an int with 1 ≤ m ≤ 65535 (the uploads kept; 1 is plain Krum).  A bool is not an int here.
    Raises ``ValueError``."""
    if isinstance(f, bool) or not isinstance(f, (int, np.integer)) or not 0 <= int(f) <= KRUM_MAX:
        raise ValueError(f"krum_f must be an int in [0, {KRUM_MAX}] (got {f!r})")
    if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 1 <= int(m) <= KRUM_MAX:
        raise ValueError(f"krum_m must be an int in [1, {KRUM_MAX}] (got {m!r})")
    return int(f), int(m)


def krum_neighbours(n: int, f: int) -> int:
    """Neighbours a Krum score sums over in a slot of n ≥ 2 uploads: clamp(n − f − 2, 1, n − 1).  Cluster sizes vary, so
    f is a per-slot assumption and every n is valid (f need not satisfy n ≥ 2f + 3)."""
    return min(max(n - f - 2, 1), n - 1)


def krum_select(D, f: int, m: int) -> Tuple[list, list]:
    """Krum scores and selection from the n × n distances ``D`` (nested lists of floats, n ≥ 2, +∞ for NaN): score_i is
    the float64 sum, from 0 in ascending order with ties by j, of the ``krum_neighbours(n, f)`` smallest D_ij over j ≠ i;
    the selection is the min(m, n) rows of smallest score (ties to the lower row, +∞ last), in ascending row order."""
    k = len(D)
    nb = krum_neighbours(k, f)
    scores = []
    for i in range(k):
        sc = 0.0
        for d, _ in sorted((D[i][j], j) for j in range(k) if j != i)[:nb]:
            sc += d
        scores.append(sc)
    return scores, sorted(sorted(range(k), key=lambda i: (scores[i], i))[:min(m, k)])


def krum_aggregate_slots_(theta: torch.Tensor, uploads: torch.Tensor, n: torch.Tensor, f: int = 1, m: int = 1,
                          mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Multi-Krum (K21; Blanchard et al., NeurIPS 2017), in place.  For every slot the participants x_1…x_n are the rows c
    with ``n[c, slot] > 0`` in ascending c, each counted once (the weights are ignored, as in ``robust_aggregate_slots_``);
    ``theta`` may be a padded bank.

    * n = 1: v is that upload.
    * Distances (n ≥ 2): D_ij = Σ_e mask_e · (double) fl32(x_ie − x_je)², the fp32 difference squared and summed in
      float64 over the trainable entries (``mask``, None = all, so BatchNorm statistics stay out); D_ij = D_ji, and a NaN
      distance counts as +∞.
    * Scores: with k = ``krum_neighbours(n, f)``, score_i is the float64 sum, from 0 in ascending order (ties by j), of the
      k smallest D_ij over j ≠ i.
    * Selection: the m_eff = min(m, n) rows of smallest score; ties go to the lower client index, +∞ ranks last.
    * Result: v_e = the fp32 sum of x_ie over the selected rows in client order, starting from the first selected value,
      then one round-to-nearest division by m_eff (none when m_eff = 1, so the slot becomes that upload bit for bit), for
      every entry (BatchNorm statistics included).

    A NaN or ±∞ row has only infinite distances, so it is never selected while enough finite rows remain; selected anyway
    (m_eff too large, or a NaN in a masked-out entry), its value propagates.  The float64 distance sums depend on the
    reduction order, so a GPU distance can differ from this one in its last bits; when no two compared scores are that
    close the selection is the same, and then the result is bit-identical (the average has a fixed order).  Slots with
    n = 0 keep θ_m.  Returns the per-slot participant counts ``[M]`` (float32)."""
    f, m_keep = krum_params(f, m)
    C, M, P = uploads.shape
    dev = uploads.device
    part = n.detach().reshape(C, M).to(dev) > 0
    counts = part.sum(0).to(torch.float32)
    keep = None if mask is None else mask.reshape(-1)[:P].to(dev, torch.bool)
    chunk = 1 << 20
    for s in range(M):
        idx = part[:, s].nonzero().flatten().tolist()
        k = len(idx)
        if k == 0:
            continue
        if k == 1:
            sel = [0]
        else:
            D = torch.zeros(k, k, dtype=torch.float64, device=dev)
            for i in range(k - 1):
                xi = uploads[idx[i], s].to(torch.float32)
                for e0 in range(0, P, chunk):
                    diff = (uploads[idx[i + 1:], s, e0:e0 + chunk].to(torch.float32) - xi[e0:e0 + chunk]).double()
                    sq = diff * diff
                    if keep is not None:
                        sq = torch.where(keep[e0:e0 + chunk], sq, torch.zeros((), dtype=torch.float64, device=dev))
                    D[i, i + 1:] += sq.sum(1)
            D = D + D.T
            D[torch.isnan(D)] = math.inf
            _, sel = krum_select(D.cpu().tolist(), f, m_keep)
        v = uploads[idx[sel[0]], s].to(torch.float32).clone()
        for i in sel[1:]:
            v = v + uploads[idx[i], s].to(torch.float32)
        if len(sel) > 1:
            v = v / torch.tensor(float(len(sel)), dtype=torch.float32, device=dev)
        theta[s, :P] = v.to(theta.device)
    return counts.to(theta.device)


CCLIP_MAX_ITERS = 100


def cclip_params(tau, iters) -> Tuple[float, int]:
    """Validated ``(--cclip_tau, --cclip_iters)``, checked whatever the rule: τ a finite number > 0 whose float32 rounding
    is finite and > 0, L an int with 1 ≤ L ≤ 100 (a bool is not a number or an int here).  Raises ``ValueError``."""
    try:
        t = None if isinstance(tau, bool) else float(tau)
    except (TypeError, ValueError):
        t = None
    if t is None or not _F32_ZERO_AT < t < _F32_INF_AT:
        raise ValueError(f"cclip_tau must be a finite number > 0 (got {tau!r})")
    if isinstance(iters, bool) or not isinstance(iters, (int, np.integer)) or not 1 <= int(iters) <= CCLIP_MAX_ITERS:
        raise ValueError(f"cclip_iters must be an int in [1, {CCLIP_MAX_ITERS}] (got {iters!r})")
    return t, int(iters)


def cclip_aggregate_slots_(theta: torch.Tensor, uploads: torch.Tensor, n: torch.Tensor, center: torch.Tensor,
                           tau: float = 1.0, iters: int = 1, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Centered clipping (K23; Karimireddy, He & Jaggi, ICML 2021), in place on ``theta`` and ``center``.  For every slot m
    the participants x_1…x_n are the rows c with ``n[c, m] > 0`` in ascending c, each counted once (the weights are
    ignored, as in ``robust_aggregate_slots_``); ``theta`` may be a padded bank, θ_m = ``theta[m, :P]`` the round-start
    model, and ``center [M, P]`` holds each slot's previous centered-clipping output h_m (the state carried from round to
    round).

    * d_ie = fl32(x_ie − θ_me) for every entry; v⁰ = h_m.
    * Iteration l = 1…L (L = ``iters``): u_ie = fl32(d_ie − v_e); r_i² = Σ_e mask_e · (double) u_ie², summed in float64
      over the trainable entries (``mask``, None = all, so BatchNorm statistics stay out); s_i = fl32(min(1, τ_f / r_i))
      computed in float64 and rounded once, τ_f = fl32(τ) widened to double (r = 0 gives 1, r = +∞ gives 0); rows with
      s_i = 0 are skipped; acc_e = Σ_i fl32(s_i · u_ie) in client order from 0, and v_e ← fl32(v_e + fl32(acc_e / n)) for
      every entry (BatchNorm statistics included).
    * θ_me ← fl32(θ_me + v_e) for every entry, and h_m ← v.

    A NaN distance makes the slot NaN (0x7FC00000) in θ_m and h_m.  The float64 distance sums depend on the reduction
    order, so the GPU matches this to a tolerance; when no row is clipped (every s_i = 1) the result is bit-identical.
    Slots with n = 0 keep θ_m and h_m.  Returns the per-slot participant counts ``[M]`` (float32)."""
    tau, L = cclip_params(tau, iters)
    tau_d = float(np.float32(tau))
    C, M, P = uploads.shape
    dev = uploads.device
    part = n.detach().reshape(C, M).to(dev) > 0
    counts = part.sum(0).to(torch.float32)
    keep = None if mask is None else mask.reshape(-1)[:P].to(dev, torch.bool)
    zero64 = torch.zeros((), dtype=torch.float64, device=dev)
    for m in range(M):
        idx = part[:, m].nonzero().flatten()
        k = int(idx.numel())
        if k == 0:
            continue
        th = theta[m, :P].to(dev, torch.float32)
        d = uploads[idx, m].to(torch.float32) - th
        v = center[m].to(dev, torch.float32).clone()
        div = torch.tensor(float(k), dtype=torch.float32, device=dev)
        nan = False
        for _ in range(L):
            u = d - v
            sq = u.double().square()
            if keep is not None:
                sq = torch.where(keep, sq, zero64)
            r2 = sq.sum(1)
            if bool(torch.isnan(r2).any()):
                nan = True
                break
            s = torch.clamp(tau_d / torch.sqrt(r2), max=1.0).to(torch.float32)
            acc = torch.zeros(P, dtype=torch.float32, device=dev)
            for i in range(k):
                if float(s[i]) != 0.0:
                    acc = acc + s[i] * u[i]
            v = v + acc / div
        if nan:
            v = torch.full((P,), _QNAN32, dtype=torch.float32, device=dev)
            theta[m, :P] = v.to(theta.device)
        else:
            theta[m, :P] = (th + v).to(theta.device)
        center[m] = v.to(center.device)
    return counts.to(theta.device)


ATTACK_TYPES = ("none", "sign_flip", "gaussian", "alie", "ipm")
_F32_ZERO_AT, _F32_INF_AT = 2.0 ** -150, 3.4028235677973366e38   # float32 rounds x ≤ the first to 0, x ≥ the second to inf
ATTACK_ID = {"none": 0, "sign_flip": 1, "gaussian": 2, "alie": 3, "ipm": 4}


def attack_params(attack_type, attack_clients, attack_scale, C: int) -> Tuple[str, int, float]:
    """Validated ``(--attack_type, --attack_clients, --attack_scale)`` of the simulated Byzantine clients, checked whatever
    the type: the type is one of ``none``, ``sign_flip``, ``gaussian``, ``alie`` or ``ipm``; a is an int with 0 ≤ a ≤ C
    (a bool is not an int here); s is a finite number > 0 whose float32 rounding is finite and > 0.  Raises
    ``ValueError``."""
    attack_type = "none" if attack_type is None else attack_type
    if attack_type not in ATTACK_TYPES:
        raise ValueError(f"attack_type must be one of {', '.join(ATTACK_TYPES)} (got {attack_type!r})")
    a = attack_clients
    if isinstance(a, bool) or not isinstance(a, (int, np.integer)) or not 0 <= int(a) <= int(C):
        raise ValueError(f"attack_clients must be an int in [0, {int(C)}] (got {a!r})")
    try:
        s = None if isinstance(attack_scale, bool) else float(attack_scale)
    except (TypeError, ValueError):
        s = None
    # float32 rounds s to a finite value > 0 exactly when 2⁻¹⁵⁰ < s < FLT_MAX + ulp/2 (plain comparisons: this runs on
    # every fused launch)
    if s is None or not _F32_ZERO_AT < s < _F32_INF_AT:
        raise ValueError(f"attack_scale must be a finite number > 0 (got {attack_scale!r})")
    return attack_type, int(a), s


def attacker_clients(C: int, a: int, seed: int) -> torch.Tensor:
    """The Byzantine clients of a run with seed ``seed`` (``--dummy_arg``): bool ``[C]``, True for the ``a`` clients with
    the smallest key mix32(seed ^ mix32(c·0x9E3779B9 + 0x85EBCA6B)), ties to the lower index.  The set is fixed for the
    run (it depends on neither the time step, the round nor client sampling) and nested in ``a``."""
    C, a = int(C), int(a)
    keys = [(mix32((seed & M32) ^ mix32((c * 0x9E3779B9 + 0x85EBCA6B) & M32)), c) for c in range(C)]
    out = torch.zeros(C, dtype=torch.bool)
    for _, c in sorted(keys)[:a]:
        out[c] = True
    return out


def attack_table(attackers, C: int, a: int) -> torch.Tensor:
    """The attacker set of ``fed_round_small``: ``attackers`` (bool/uint8 [C]) when given, which must hold exactly ``a``
    clients, else ``attacker_clients(C, a, 0)``.  Raises ``ValueError``."""
    if attackers is None:
        return attacker_clients(C, a, 0)
    att = torch.as_tensor(attackers).detach().cpu().reshape(-1).bool()
    if att.numel() != int(C) or int(att.sum()) != int(a):
        raise ValueError(f"attackers must be a [C = {int(C)}] table of exactly attack_clients = {int(a)} clients")
    return att


def attack_seed(seed: int, rnd: int) -> int:
    """``gauss_hash`` seed of the ``gaussian`` attack in round ``rnd`` of a time step whose engine seed is ``seed`` (the
    ``attack_seed`` of csrc/common.cuh): a function of (seed, round) only, with constants that differ from those of
    ``defense_seed`` and ``compress_seed``."""
    return mix32((seed & M32) ^ mix32((rnd * 0x85EBCA77 + 0x3C6EF372) & M32))


def attack_slots_(rows: torch.Tensor, theta: torch.Tensor, n, attackers, attack_type: str, scale: float,
                  weight_mask=None, seed: int = 0) -> torch.Tensor:
    """Model poisoning (K22) of an upload arena ``rows [C, M, P]``, in place.  For every slot m, with θ = ``theta[m, :P]``
    (``theta`` may be a padded bank) and s = fl32(``scale``), every attacker pair (``attackers[c]``, ``n[c, m] > 0``)
    uploads, on each entry e with ``weight_mask`` True (None = all; BatchNorm statistics keep the attacker's values):

    * ``sign_flip``: θ − fl32(s·fl32(x − θ)), its own update reversed and scaled by s;
    * ``gaussian``: θ + fl32(s·ξ), ξ = ``gauss_hash(seed, c·M + m, e)``;
    * ``alie``: μ − fl32(s·σ) (A Little Is Enough, Baruch et al. 2019; s is their z);
    * ``ipm``: θ − fl32(s·fl32(μ − θ)) (inner-product manipulation, Xie et al. 2019; s is their ε).

    μ is the fp32 sum, from 0 in client order, of the honest uploads of the slot (c not an attacker, n[c, m] > 0), divided
    once by their number h; σ = sqrt_rn(fl32(Σ fl32(δ·δ)) / h) with δ = fl32(x − μ), summed from 0 in client order (the
    population standard deviation).  Every operation is rounded on its own.  The attackers of a slot collude under
    ``alie`` and ``ipm``: they upload the same vector; with h = 0 their rows are left as trained.  Pairs with n ≤ 0 and
    honest pairs are untouched.  Returns ``rows``."""
    C, M, P = rows.shape
    attack_type, _, scale = attack_params(attack_type, 0, scale, C)
    if attack_type == "none" or C * M == 0 or P == 0:
        return rows
    dev = rows.device
    th = theta[:, :P].to(dev, torch.float32)
    sel = torch.ones(C, M, dtype=torch.bool) if n is None else (n.detach().cpu().reshape(C, M) > 0)
    att = torch.as_tensor(attackers).detach().cpu().reshape(-1).bool()
    if att.numel() != C:
        raise ValueError(f"attack_slots_: attackers must have C = {C} entries (got {att.numel()})")
    wm = None if weight_mask is None else weight_mask.reshape(-1)[:P].to(dev).bool()
    sf = torch.tensor(scale, dtype=torch.float32, device=dev)
    for m in range(M):
        bad = [c for c in range(C) if bool(att[c]) and bool(sel[c, m])]
        if not bad:
            continue
        if attack_type in ("alie", "ipm"):
            good = [c for c in range(C) if not bool(att[c]) and bool(sel[c, m])]
            if not good:
                continue
            hf = torch.tensor(float(len(good)), dtype=torch.float32, device=dev)
            acc = torch.zeros(P, dtype=torch.float32, device=dev)
            for c in good:
                acc = acc + rows[c, m]
            mu = acc / hf
            if attack_type == "alie":
                ss = torch.zeros(P, dtype=torch.float32, device=dev)
                for c in good:
                    d = rows[c, m] - mu
                    ss = ss + d * d
                # sqrt_rn: the float64 root of a float32 rounds to the correctly rounded float32 root (torch's float32
                # CPU sqrt is not always correctly rounded)
                crafted = mu - sf * torch.sqrt((ss / hf).double()).float()
            else:
                crafted = th[m] - sf * (mu - th[m])
        for c in bad:
            row = rows[c, m]
            if attack_type == "sign_flip":
                new = th[m] - sf * (row - th[m])
            elif attack_type == "gaussian":
                new = th[m] + sf * gauss_hash_rows(seed, [c * M + m], P)[0].to(dev)
            else:
                new = crafted
            row.copy_(new if wm is None else torch.where(wm, new, row))
    return rows


def server_opt_step_(theta, avg, state: Dict, opt: str, lr: float, momentum=0.0, b1=0.9, b2=0.999, eps=1e-8):
    """FedOpt (K11): pseudo-gradient g = theta - avg, then one server-optimizer step in place."""
    g = theta - avg
    if opt == "sgd":
        if momentum:
            buf = state.setdefault("momentum", torch.zeros_like(theta))
            buf.mul_(momentum).add_(g)
            g = buf
        theta.add_(g, alpha=-lr)
    elif opt == "adam":
        state["step"] = state.get("step", 0) + 1
        m = state.setdefault("m", torch.zeros_like(theta))
        v = state.setdefault("v", torch.zeros_like(theta))
        m.mul_(b1).add_(g, alpha=1 - b1)
        v.mul_(b2).addcmul_(g, g, value=1 - b2)
        bc1, bc2 = 1 - b1 ** state["step"], 1 - b2 ** state["step"]
        theta.addcdiv_(m, v.sqrt() / math.sqrt(bc2) + eps, value=-lr / bc1)
    elif opt == "adagrad":
        s = state.setdefault("sum", torch.zeros_like(theta))
        s.addcmul_(g, g)
        theta.addcdiv_(g, s.sqrt() + eps, value=-lr)
    elif opt == "yogi":
        state["step"] = state.get("step", 0) + 1
        m = state.setdefault("m", torch.zeros_like(theta))
        v = state.setdefault("v", torch.full_like(theta, 1e-6))
        m.mul_(b1).add_(g, alpha=1 - b1)
        g2 = g * g
        v.sub_((1 - b2) * torch.sign(v - g2) * g2)
        theta.addcdiv_(m, v.sqrt() + eps, value=-lr)
    else:
        raise ValueError(opt)
    return theta


_SLOT_STATE_KEYS = {"sgd": ("momentum", None), "adam": ("m", "v"), "adagrad": ("sum", None), "yogi": ("m", "v")}


def server_opt_slots_(theta, avg, active, opt: str, s0, s1, steps, lr: float, momentum: float = 0.0, eps: float = 1e-8,
                      mask=None) -> None:
    """Per-slot FedOpt step, in place: for every slot m with ``active[m]``, θ_m takes one ``server_opt_step_`` on
    θ_m − avg_m with the slot's own state rows ``s0[m]`` / ``s1[m]`` (None where ``opt`` has no such state) and its own step
    count ``steps[m]`` (Adam's bias correction uses steps[m] + 1), then ``steps[m]`` advances.  Entries with ``mask`` False
    take avg_m and keep their state.  Inactive slots are left untouched."""
    k0, k1 = _SLOT_STATE_KEYS[opt]
    sel = torch.ones(theta.shape[1], dtype=torch.bool, device=theta.device) if mask is None else mask.to(theta.device, torch.bool)
    for m in range(theta.shape[0]):
        if not bool(active[m]):
            continue
        th = theta[m, sel]
        state = {"step": int(steps[m])}
        if s0 is not None:
            state[k0] = s0[m, sel]
        if s1 is not None:
            state[k1] = s1[m, sel]
        server_opt_step_(th, avg[m, sel], state, opt, lr, momentum=momentum, eps=eps)
        theta[m, sel] = th
        if s0 is not None:
            s0[m, sel] = state[k0]
        if s1 is not None:
            s1[m, sel] = state[k1]
        if mask is not None:
            theta[m, ~sel] = avg[m, ~sel]
        steps[m] += 1


def ada_stats(theta: torch.Tensor, prev_muh: torch.Tensor) -> float:
    """mean((θ - μ̂_{t-1})²) — the only O(P) term of Adaptive-FedAvg's LR rule (K8)."""
    return float(((theta - prev_muh) ** 2).mean())


def gossip_mix(X: torch.Tensor, Wmix: torch.Tensor) -> torch.Tensor:
    """x_i <- Σ_j W_ij x_j over rows (K12)."""
    return Wmix.to(X.dtype) @ X


def merge_axpby_(theta: torch.Tensor, base: int, second: int, w1: float, w2: float) -> None:
    theta[base] = theta[base] * w1 + theta[second] * w2


# --------------------------------------------------------------------------- K4 / K7 (big models: from logits)
def eval_logits(logits: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """-> tensor [3] (correct, loss_sum, count) accumulated on device, no host sync."""
    loss = F.cross_entropy(logits.float(), target.long(), reduction="sum")
    correct = (logits.argmax(-1) == target).sum()
    return torch.stack([correct.float(), loss.float(), torch.tensor(float(target.numel()), device=logits.device)])


def aue_sqerr(logits: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """Σ (1 - softmax(logits)[y])²  (AUE MSE_i numerator)."""
    p = F.softmax(logits.float(), dim=1).gather(1, target.long()[:, None]).squeeze(1)
    return ((1.0 - p) ** 2).sum()


def ensemble_vote(preds: torch.Tensor, weights: torch.Tensor, num_classes: int) -> torch.Tensor:
    """preds [K,B] int hard votes, weights [K] -> argmax_c Σ_k w_k·[pred_k == c]  ([B])."""
    K, B = preds.shape
    tally = torch.zeros(B, num_classes, dtype=torch.float64, device=preds.device)
    for k in range(K):
        tally[torch.arange(B, device=preds.device), preds[k].long()] += float(weights[k])
    return tally.argmax(-1)


def soft_vote(probs: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
    """probs [K,B,C], weights [K] (≤0 entries skipped) -> argmax Σ w_k p_k  (KUE)."""
    w = torch.clamp(weights.to(probs.dtype), min=0)
    return (probs * w[:, None, None]).sum(0).argmax(-1)


def confusion_matrix(pred: torch.Tensor, target: torch.Tensor, num_classes: int) -> torch.Tensor:
    idx = target.long() * num_classes + pred.long()
    return torch.bincount(idx, minlength=num_classes * num_classes).reshape(num_classes, num_classes).double()


def cohen_kappa(A: torch.Tensor) -> float:
    n = float(A.sum())
    left = float(torch.diagonal(A).sum())
    right = float((A.sum(1) * A.sum(0)).sum())
    den = n * n - right
    return (n * left - right) / den if den != 0 else 0.0


# --------------------------------------------------------------------------- K5 / K6
def cluster_distance(acc: np.ndarray, kind: str = "A") -> np.ndarray:
    """FedDrift cluster distance from the L×L cross-accuracy matrix (a_ij = acc of model i on data j)."""
    a = np.asarray(acc, dtype=np.float64)
    d = np.diag(a)
    if kind == "A":
        D = np.maximum(d[:, None] - a, (d[:, None] - a).T)
    else:
        D = np.maximum(d[:, None] - a.T, (d[:, None] - a.T).T)
    return np.maximum(D, 0.0)


def gram_cosine(U: torch.Tensor, eps: float = 1e-12):
    """U [n,P] -> (cosine-similarity [n,n], norms [n])  (CFL, K6)."""
    G = U.double() @ U.double().t()
    nrm = torch.sqrt(torch.diagonal(G))
    return (G / (nrm[:, None] * nrm[None, :] + eps)), nrm


# --------------------------------------------------------------------------- K13..K16
def modp_matmul(A: torch.Tensor, B: torch.Tensor, p: int) -> torch.Tensor:
    """(A @ B) mod p, exact for any p < 2**63 (python-int arithmetic when products could overflow int64)."""
    A, B = A.to(torch.int64) % p, B.to(torch.int64) % p
    if p < (1 << 31):
        out = torch.zeros(A.shape[0], B.shape[1], dtype=torch.int64)
        for k in range(A.shape[1]):  # products < 2^62: reduce per term
            out = (out + (A[:, k:k + 1] * B[k:k + 1, :]) % p) % p
        return out
    An, Bn = A.numpy().astype(object), B.numpy().astype(object)
    return torch.from_numpy((An.dot(Bn) % p).astype(np.int64))


def kd_kl_loss(student_logits, teacher_logits, temperature: float = 1.0):
    """FedGKT distillation loss: T² · KL(softmax(t/T) ‖ softmax(s/T)), batch-mean (K14)."""
    T = temperature
    ls = F.log_softmax(student_logits / T, dim=1)
    pt = F.softmax(teacher_logits / T, dim=1) + 1e-7
    return (T * T) * (pt * (torch.log(pt) - ls)).sum(1).mean()


def vfl_bce_grad(logit_parts: torch.Tensor, y: torch.Tensor):
    """logit_parts [K,B,1] -> (mean BCE-with-logits loss, dL/dlogit [B,1]) for the summed logit (K15)."""
    z = logit_parts.sum(0)
    loss = F.binary_cross_entropy_with_logits(z, y.float(), reduction="mean")
    grad = (torch.sigmoid(z) - y.float()) / z.shape[0]
    return loss, grad


def group_norm(x: torch.Tensor, groups: int, weight=None, bias=None, eps: float = 1e-5):
    return F.group_norm(x, groups, weight, bias, eps)
