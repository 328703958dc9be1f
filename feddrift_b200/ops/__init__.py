"""Op surface of the framework.  Every function dispatches to the hand-written
sm_90a kernel when its tensors live on CUDA (the extension is then mandatory)
and to the fp32 PyTorch reference (``ops.reference``) on CPU.

Kernel map (SURVEY §2.9 numbering):
  K1  cluster_aggregate_ / weighted_average      csrc/aggregate.cu
  K3  fed_round_small (fused local step+K1+K4)    csrc/fed_round_small.cu
      adam_amsgrad_rows_ (arena optimizer)        csrc/optim.cu
      TcLinear GEMM (wgmma/TMA)            csrc/gemm_tc.cu
  K4  mlp_eval_matrix / eval_logits_              csrc/eval.cu
  K5  merge_axpby_ / cluster_distance             csrc/aggregate.cu / host (L ≤ #models)
  K6  gram_cosine                                 csrc/cluster_ops.cu
  K7  aue_sqerr / ensemble_vote / confusion       csrc/eval.cu
  K8  ada_stats (fused mean-square)               csrc/aggregate.cu
  K10 robust_clip_ / robust_clip_slots_           csrc/aggregate.cu
  K11 server_opt_step_                            csrc/aggregate.cu
  K12 gossip_mix                                  csrc/aggregate.cu
  K13 modp_matmul                                 csrc/mpc.cu
  K14 kd_kl_loss   K15 vfl_bce_grad   K16 group_norm   csrc/misc.cu
  K17 qsgd_slots_ (upload quantization)           csrc/compress.cu
  K18 eftopk_slots_ (top-k + error feedback)      csrc/sparsify.cu
  K19 robust_aggregate_slots_ (median / trimmed mean)   csrc/robust_agg.cu
  K20 geomed_aggregate_slots_ (geometric median)        csrc/robust_agg.cu
  K21 krum_aggregate_slots_ (Multi-Krum)                csrc/robust_agg.cu
  K22 attack_slots_ (simulated Byzantine clients)       csrc/attack.cu
  K23 cclip_aggregate_slots_ (centered clipping)        csrc/robust_agg.cu
"""
from __future__ import annotations

from typing import Dict

import torch

from . import _ext, reference as ref
from .reference import (batch_hash, cluster_distance, cohen_kappa, hash_choice, mix32, mlp_forward,  # noqa: F401
                        mlp_param_count, mlp_unpack)

KIND_ID = {"lr": 0, "fnn": 1}
OPT_ID = {"sgd": 0, "adam": 1}


def native(*tensors) -> bool:
    return _ext.use_native(*tensors)


# ----------------------------------------------------------------------------- K3 fused small round
def fed_round_small(st: Dict, rounds: int = 1) -> Dict[str, torch.Tensor]:
    """Run ``rounds`` complete FL rounds (broadcast → local steps → per-cluster aggregate →
    optional IFCA re-cluster → train/test evaluation of every client) for a small-MLP federation.
    See ``reference.fed_round_small`` for the exact semantics."""
    if native(st["theta"]):
        from .small_round import run_native
        return run_native(st, rounds)
    return ref.fed_round_small(st, rounds)


# ----------------------------------------------------------------------------- K1
def cluster_aggregate_(theta, client_params, n, server_opt=None, rule=None, mask=None, center=None):
    """K1: θ_m ← weighted mean of ``client_params[:, m]`` for every slot with total weight > 0; returns the totals [M].
    ``server_opt`` (``server_opt.SlotServerOpt``) then steps each such slot on θ_m − avg_m with its own state.
    ``rule`` = ``(aggregation_rule, trim_ratio)`` with rule 'median' or 'trimmed_mean' replaces the weighted mean by K19
    (``robust_aggregate_slots_``: the participants n > 0 count once each) and returns the participant counts [M]; None or
    'mean' is the weighted mean above.  ``rule`` = ``('geometric_median', trim_ratio, iters, nu)`` takes K20
    (``geomed_aggregate_slots_``) instead, with ``mask`` the trainable entries its distances cover (None: all), and
    ``('multi_krum', trim_ratio, f, m)`` takes K21 (``krum_aggregate_slots_``) with the same ``mask``.
    ``('centered_clip', trim_ratio, tau, iters)`` takes K23 (``cclip_aggregate_slots_``) with the same ``mask`` around
    ``center`` [M, P], the slots' state, which it updates; it is required for this rule and ignored otherwise."""
    if rule is not None and rule[0] == "centered_clip":
        if center is None:
            raise ValueError("cluster_aggregate_: centered_clip needs the slots' centers (center=)")
        return cclip_aggregate_slots_(theta, client_params, n, center, rule[2], rule[3], server_opt, mask)
    if rule is not None and rule[0] == "geometric_median":
        return geomed_aggregate_slots_(theta, client_params, n, rule[2], rule[3], server_opt, mask)
    if rule is not None and rule[0] == "multi_krum":
        return krum_aggregate_slots_(theta, client_params, n, rule[2], rule[3], server_opt, mask)
    if rule is not None and rule[0] != "mean":
        return robust_aggregate_slots_(theta, client_params, n, rule[0], rule[1], server_opt)
    if server_opt is not None:
        if native(theta, client_params):
            return server_opt.aggregate_native_(theta, client_params, n)
        return server_opt.aggregate_reference_(theta, client_params, n)
    if native(theta, client_params):
        return _ext.load().cluster_aggregate(theta, client_params.contiguous(), n.float().contiguous())
    return ref.cluster_aggregate_(theta, client_params, n)


def robust_aggregate_slots_(theta, uploads, n, rule: str = "median", trim_ratio: float = 0.1, server_opt=None):
    """K19: θ_m ← coordinate-wise median / trimmed mean of the uploads ``uploads[c, m]`` with ``n[c, m] > 0`` (each counted
    once) for every slot with a participant; ``theta`` may be a padded bank.  ``server_opt`` (``server_opt.SlotServerOpt``)
    then steps each such slot on θ_m − statistic and advances its counter.  See ``reference.robust_aggregate_slots_``;
    returns the participant counts [M]."""
    rule, beta = ref.aggregation_params(rule, trim_ratio)
    if rule not in ("median", "trimmed_mean"):
        raise ValueError("robust_aggregate_slots_: rule must be median or trimmed_mean")
    if native(theta, uploads):
        rid = 1 if rule == "median" else 2
        nn = n.float().contiguous()
        if server_opt is None:
            return _ext.load().robust_aggregate_slots(theta, uploads.contiguous(), nn, rid, beta, 0, 0.0, 0.0, 1e-8,
                                                      None, None, None, None)
        so = server_opt
        return _ext.load().robust_aggregate_slots(theta, uploads.contiguous(), nn, rid, beta, so.kind, so.lr, so.momentum, so.eps,
                                                  so.s0, so.s1, so.step, so._mask_u8)
    if server_opt is None:
        return ref.robust_aggregate_slots_(theta, uploads, n, rule, beta)
    avg = theta.clone()
    counts = ref.robust_aggregate_slots_(avg, uploads, n, rule, beta)
    so = server_opt
    ref.server_opt_slots_(theta, avg, counts > 0, so.opt, so.s0, so.s1, so.step, so.lr, so.momentum, so.eps, so.mask)
    return counts


def geomed_aggregate_slots_(theta, uploads, n, iters: int = 4, nu: float = 1e-6, server_opt=None, mask=None):
    """K20: θ_m ← geometric median (``iters`` smoothed Weiszfeld steps from the coordinate-wise median, smoothing ``nu``) of
    the uploads ``uploads[c, m]`` with ``n[c, m] > 0`` (each counted once) for every slot with a participant; ``theta`` may be
    a padded bank; ``mask`` [P] (bool, None = all) selects the entries of the distances (BatchNorm statistics are
    aggregated but left out).  ``server_opt`` then steps each such slot on θ_m − v and advances its counter.  See
    ``reference.geomed_aggregate_slots_``; returns the participant counts [M]."""
    iters, nu = ref.geomed_params(iters, nu)
    if native(theta, uploads):
        nn = n.float().contiguous()
        dm = None if mask is None else mask.reshape(-1)[: uploads.shape[2]].to(uploads.device, torch.uint8).contiguous()
        if server_opt is None:
            return _ext.load().geomed_aggregate_slots(theta, uploads.contiguous(), nn, iters, nu, 0, 0.0, 0.0, 1e-8,
                                                      None, None, None, None, dm)
        so = server_opt
        return _ext.load().geomed_aggregate_slots(theta, uploads.contiguous(), nn, iters, nu, so.kind, so.lr, so.momentum, so.eps,
                                                  so.s0, so.s1, so.step, so._mask_u8, dm)
    if server_opt is None:
        return ref.geomed_aggregate_slots_(theta, uploads, n, iters, nu, mask)
    avg = theta.clone()
    counts = ref.geomed_aggregate_slots_(avg, uploads, n, iters, nu, mask)
    so = server_opt
    ref.server_opt_slots_(theta, avg, counts > 0, so.opt, so.s0, so.s1, so.step, so.lr, so.momentum, so.eps, so.mask)
    return counts


def krum_aggregate_slots_(theta, uploads, n, f: int = 1, m: int = 1, server_opt=None, mask=None):
    """K21: θ_s ← Multi-Krum of the uploads ``uploads[c, s]`` with ``n[c, s] > 0`` (each counted once) for every slot with
    a participant: the average of the min(``m``, n) uploads whose summed squared distances to their clamp(n − ``f`` − 2, 1,
    n − 1) nearest neighbours are smallest (``m`` = 1: plain Krum, the slot becomes one upload); ``theta`` may be a padded
    bank; ``mask`` [P] (bool, None = all) selects the entries of the distances (BatchNorm statistics are averaged but left
    out).  ``server_opt`` then steps each such slot on θ_s − v and advances its counter.  See
    ``reference.krum_aggregate_slots_``; returns the participant counts [M]."""
    f, m = ref.krum_params(f, m)
    if native(theta, uploads):
        nn = n.float().contiguous()
        dm = None if mask is None else mask.reshape(-1)[: uploads.shape[2]].to(uploads.device, torch.uint8).contiguous()
        if server_opt is None:
            return _ext.load().krum_aggregate_slots(theta, uploads.contiguous(), nn, f, m, 0, 0.0, 0.0, 1e-8,
                                                    None, None, None, None, dm)
        so = server_opt
        return _ext.load().krum_aggregate_slots(theta, uploads.contiguous(), nn, f, m, so.kind, so.lr, so.momentum, so.eps,
                                                so.s0, so.s1, so.step, so._mask_u8, dm)
    if server_opt is None:
        return ref.krum_aggregate_slots_(theta, uploads, n, f, m, mask)
    avg = theta.clone()
    counts = ref.krum_aggregate_slots_(avg, uploads, n, f, m, mask)
    so = server_opt
    ref.server_opt_slots_(theta, avg, counts > 0, so.opt, so.s0, so.s1, so.step, so.lr, so.momentum, so.eps, so.mask)
    return counts


def cclip_aggregate_slots_(theta, uploads, n, center, tau: float = 1.0, iters: int = 1, server_opt=None, mask=None):
    """K23: θ_m ← θ_m + v_m, centered clipping (``iters`` steps of radius ``tau`` around the slot's center, its previous
    output) of the updates ``uploads[c, m]`` − θ_m with ``n[c, m] > 0`` (each counted once) for every slot with a
    participant, and ``center[m]`` ← v_m; ``theta`` may be a padded bank; ``mask`` [P] (bool, None = all) selects the
    entries of the distances (BatchNorm statistics are clipped along but left out).  ``server_opt`` then steps each such
    slot on θ_m − (θ_m + v_m) and advances its counter.  See ``reference.cclip_aggregate_slots_``; returns the participant
    counts [M]."""
    tau, iters = ref.cclip_params(tau, iters)
    if native(theta, uploads):
        nn = n.float().contiguous()
        dm = None if mask is None else mask.reshape(-1)[: uploads.shape[2]].to(uploads.device, torch.uint8).contiguous()
        if server_opt is None:
            return _ext.load().cclip_aggregate_slots(theta, uploads.contiguous(), nn, center, tau, iters, 0, 0.0, 0.0, 1e-8,
                                                     None, None, None, None, dm)
        so = server_opt
        return _ext.load().cclip_aggregate_slots(theta, uploads.contiguous(), nn, center, tau, iters, so.kind, so.lr, so.momentum,
                                                 so.eps, so.s0, so.s1, so.step, so._mask_u8, dm)
    if server_opt is None:
        return ref.cclip_aggregate_slots_(theta, uploads, n, center, tau, iters, mask)
    avg = theta.clone()
    counts = ref.cclip_aggregate_slots_(avg, uploads, n, center, tau, iters, mask)
    so = server_opt
    ref.server_opt_slots_(theta, avg, counts > 0, so.opt, so.s0, so.s1, so.step, so.lr, so.momentum, so.eps, so.mask)
    return counts


def weighted_average(rows, weights, out=None):
    if native(rows):
        res = _ext.load().weighted_average(rows.contiguous(), weights.float().contiguous())
    else:
        res = ref.weighted_average(rows, weights)
    if out is not None:
        out.copy_(res)
        return out
    return res


def robust_clip_(rows, global_row, bound: float, weight_mask=None, stddev: float = 0.0, seed: int = 0):
    """K10: clip every row around ``global_row`` and (``stddev > 0``) add counter-hash Gaussian noise in the same pass."""
    if native(rows):
        mask = weight_mask.to(torch.uint8).contiguous() if weight_mask is not None else None
        return _ext.load().robust_clip(rows, global_row.contiguous(), float(bound), mask, float(stddev), int(seed) & 0xFFFFFFFF)
    return ref.robust_clip_(rows, global_row, bound, weight_mask, stddev, seed)


def robust_clip_slots_(rows, theta, n=None, bound: float = 5.0, weight_mask=None, stddev: float = 0.0, seed: int = 0):
    """K10 over an upload arena ``rows [C, M, P]``: every row with ``n[c, m] > 0`` is clipped around its slot's model
    ``theta[m, :P]`` (``theta`` may be a padded bank) and, with ``stddev > 0``, gets ``gauss_hash(seed, c·M + m, ·)`` noise.
    See ``reference.robust_clip_slots_``; returns the norms ``[C, M]``."""
    if native(rows, theta):
        mask = weight_mask[: rows.shape[2]].to(torch.uint8).contiguous() if weight_mask is not None else None
        nn = n.float().contiguous() if n is not None else None
        out = _ext.load().robust_clip_slots(rows, theta, nn, float(bound), mask, float(stddev), int(seed) & 0xFFFFFFFF)
        return out.view(rows.shape[0], rows.shape[1])
    return ref.robust_clip_slots_(rows, theta, n, bound, weight_mask, stddev, seed)


def qsgd_slots_(rows, theta, n=None, level: int = 16, bucket: int = 512, weight_mask=None, seed: int = 0):
    """K17: QSGD of an upload arena ``rows [C, M, P]`` in place: every row with ``n[c, m] > 0`` is quantized against its
    slot's model ``theta[m, :P]`` (``theta`` may be a padded bank) with level ``level`` and bucket ``bucket``; the draws are
    ``uniform_hash(seed, c·M + m, ·)``.  See ``reference.qsgd_slots_``; returns ``rows``."""
    if native(rows, theta):
        mask = weight_mask[: rows.shape[2]].to(torch.uint8).contiguous() if weight_mask is not None else None
        nn = n.float().contiguous() if n is not None else None
        _ext.load().qsgd_slots(rows, theta, nn, int(level), int(bucket), mask, int(seed) & 0xFFFFFFFF)
        return rows
    return ref.qsgd_slots_(rows, theta, n, level, bucket, weight_mask, seed)


def eftopk_slots_(rows, theta, residual, n=None, k: int = 1, weight_mask=None):
    """K18: top-k with error feedback of an upload arena ``rows [C, M, P]`` and its residual ``residual [C, M, P]``, in
    place: every row with ``n[c, m] > 0`` keeps its ``k`` largest error-corrected entries against its slot's model
    ``theta[m, :P]`` (``theta`` may be a padded bank) and carries the rest in the residual.  See
    ``reference.eftopk_slots_``; returns ``rows``."""
    if native(rows, theta, residual):
        mask = weight_mask[: rows.shape[2]].to(torch.uint8).contiguous() if weight_mask is not None else None
        nn = n.float().contiguous() if n is not None else None
        _ext.load().eftopk_slots(rows, theta, residual, nn, int(k), mask)
        return rows
    return ref.eftopk_slots_(rows, theta, residual, n, k, weight_mask)


def attack_slots_(rows, theta, n, attackers, kind: str, scale: float = 1.0, mask=None, seed: int = 0):
    """K22: simulated Byzantine clients of an upload arena ``rows [C, M, P]`` in place: every pair of a client with
    ``attackers[c]`` (bool [C]) and ``n[c, m] > 0`` uploads the poisoned value of ``kind`` ('sign_flip', 'gaussian' with
    noise ``gauss_hash(seed, c·M + m, ·)``, 'alie' or 'ipm') with strength ``scale`` against its slot's model
    ``theta[m, :P]`` (``theta`` may be a padded bank) on the entries of ``mask`` (bool [P], None = all).  'none' is a
    no-op.  See ``reference.attack_slots_``; returns ``rows``."""
    kind, _, scale = ref.attack_params(kind, 0, scale, rows.shape[0])
    if kind == "none":
        return rows
    if native(rows, theta):
        dev = rows.device
        att = torch.as_tensor(attackers).reshape(-1).to(dev, torch.uint8).contiguous()
        dm = None if mask is None else mask.reshape(-1)[: rows.shape[2]].to(dev, torch.uint8).contiguous()
        _ext.load().attack_slots(rows, theta, n.float().contiguous(), att, ref.ATTACK_ID[kind], scale, dm,
                                 int(seed) & 0xFFFFFFFF)
        return rows
    return ref.attack_slots_(rows, theta, n, attackers, kind, scale, mask, seed)


def server_opt_step_(theta, avg, state: Dict, opt: str, lr: float, **kw):
    if native(theta) and opt in ("sgd", "adam", "adagrad", "yogi"):
        from .server_opt import native_server_opt_step_
        return native_server_opt_step_(theta, avg, state, opt, lr, **kw)
    return ref.server_opt_step_(theta, avg, state, opt, lr, **kw)


def ada_stats(theta, prev_muh) -> float:
    if native(theta):
        return float(_ext.load().mean_sq_diff(theta.contiguous(), prev_muh.contiguous()))
    return ref.ada_stats(theta, prev_muh)


def gossip_mix(X, Wmix):
    if native(X):
        return _ext.load().gossip_mix(X.contiguous(), Wmix.float().contiguous())
    return ref.gossip_mix(X, Wmix)


def merge_axpby_(theta, base: int, second: int, w1: float, w2: float):
    if native(theta):
        _ext.load().merge_axpby(theta, int(base), int(second), float(w1), float(w2))
    else:
        ref.merge_axpby_(theta, base, second, w1, w2)


# ----------------------------------------------------------------------------- K4 / K7
def mlp_eval_matrix(theta, X, Y, nsamp, kind, din, hid, dout):
    if native(theta, X):
        out = _ext.load().mlp_eval_matrix(theta.contiguous(), X.contiguous(), Y.int().contiguous(),
                                          nsamp.int().contiguous(), KIND_ID[kind], din, hid, dout)
        return out[0], out[1]
    return ref.mlp_eval_matrix(theta, X, Y, nsamp, kind, din, hid, dout)


def eval_logits(logits, target, acc=None):
    """Accumulate (correct, loss_sum, count) into ``acc`` [3] on device without a host sync."""
    if native(logits):
        if acc is None:
            acc = torch.zeros(3, dtype=torch.float32, device=logits.device)
        _ext.load().eval_logits(logits.float().contiguous(), target.int().contiguous(), acc)
        return acc
    r = ref.eval_logits(logits, target)
    if acc is not None:
        acc += r
        return acc
    return r


def aue_sqerr(logits, target):
    if native(logits):
        return _ext.load().aue_sqerr(logits.float().contiguous(), target.int().contiguous())
    return ref.aue_sqerr(logits, target)


def ensemble_vote(preds, weights, num_classes: int):
    if native(preds):
        return _ext.load().ensemble_vote(preds.int().contiguous(), weights.float().contiguous(), int(num_classes))
    return ref.ensemble_vote(preds, weights, num_classes)


def soft_vote(probs, weights):
    return ref.soft_vote(probs, weights)


def confusion_matrix(pred, target, num_classes: int):
    if native(pred):
        return _ext.load().confusion_matrix(pred.int().contiguous(), target.int().contiguous(),
                                            int(num_classes)).double()
    return ref.confusion_matrix(pred, target, num_classes)


# ----------------------------------------------------------------------------- K6
def gram_cosine(U, eps: float = 1e-12):
    if native(U):
        out = _ext.load().gram_cosine(U.float().contiguous(), float(eps))
        return out[0], out[1]
    return ref.gram_cosine(U, eps)


# ----------------------------------------------------------------------------- arena optimizer
def _prox_args(prox):
    """``prox=(mu, anchor, anchor_rows, mask)`` → the trailing arguments of the native row optimizers (no anchor: off)."""
    if prox is None:
        return 0.0, None, None, None
    mu, anchor, rows, mask = prox
    return float(mu), anchor, rows, mask


def adam_amsgrad_rows_(p, g, m, v, vmax, steps, lr: float, wd: float, b1=0.9, b2=0.999, eps=1e-8, row_mask=None, prox=None):
    """Fused Adam(amsgrad, L2 wd) over arena rows [R,P]; ``steps`` [R] int32 is incremented in place.  ``prox=(mu, anchor,
    anchor_rows, mask)`` adds the FedProx term mu·mask⊙(p[r] − anchor[anchor_rows[r]]) to row r's gradient before the wd term
    (``reference.prox_grad``): anchor [A, ≥ P] with unit column stride, anchor_rows int32 [R], mask uint8 [P] or None.  With
    ``prox``, the updated rows of ``g`` are overwritten by that effective gradient (g must be contiguous)."""
    if native(p):
        _ext.load().adam_amsgrad_rows(p, g if prox is not None else g.contiguous(), m, v, vmax, steps, float(lr), float(wd), float(b1),
                                      float(b2), float(eps), row_mask, *_prox_args(prox))
        return p
    for r in range(p.shape[0]):
        if row_mask is not None and not bool(row_mask[r]):
            continue
        if prox is not None:
            g[r] = ref.prox_grad(g[r], p[r], prox, r)
        steps[r] = ref.adam_amsgrad_update(p[r], g[r], m[r], v[r], vmax[r], int(steps[r]), lr, wd, b1, b2, eps)
    return p


def sgd_rows_(p, g, lr: float, wd: float = 0.0, row_mask=None, prox=None):
    """p ← p − lr·(g + wd·p) over arena rows [R,P]; ``row_mask`` uint8 [R] skips rows, ``prox`` as in ``adam_amsgrad_rows_``."""
    if native(p):
        _ext.load().sgd_rows(p, g.contiguous(), float(lr), float(wd), row_mask, *_prox_args(prox))
        return p
    if row_mask is None and prox is None:
        p.add_(g + wd * p, alpha=-lr)
        return p
    for r in range(p.shape[0]):
        if row_mask is not None and not bool(row_mask[r]):
            continue
        gr = g[r] if prox is None else ref.prox_grad(g[r], p[r], prox, r)
        p[r].add_(gr + wd * p[r], alpha=-lr)
    return p


# ----------------------------------------------------------------------------- K13..K16
def modp_matmul(A, B, p: int):
    if native(A):
        return _ext.load().modp_matmul(A.long().contiguous(), B.long().contiguous(), int(p))
    return ref.modp_matmul(A, B, p)


class _KDLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s, t, T):
        out = _ext.load().kd_kl_fwd_bwd(s.float().contiguous(), t.float().contiguous(), float(T))
        ctx.save_for_backward(out[1])
        return out[0]

    @staticmethod
    def backward(ctx, g):
        (gs,) = ctx.saved_tensors
        return gs * g, None, None


def kd_kl_loss(student_logits, teacher_logits, temperature: float = 1.0):
    if native(student_logits):
        return _KDLoss.apply(student_logits, teacher_logits.detach(), temperature)
    return ref.kd_kl_loss(student_logits, teacher_logits, temperature)


def vfl_bce_grad(logit_parts, y):
    if native(logit_parts):
        out = _ext.load().vfl_bce_grad(logit_parts.float().contiguous(), y.float().contiguous())
        return out[0], out[1]
    return ref.vfl_bce_grad(logit_parts, y)


class _GroupNormFn(torch.autograd.Function):
    """K16 with autograd: fused forward (saves per-group mean / rstd) + fused backward kernel (csrc/misc.cu)."""

    @staticmethod
    def forward(ctx, x, weight, bias, groups, eps):
        xc = x.float().contiguous()
        y, mean, rstd = _ext.load().group_norm_fwd_train(xc, int(groups), weight, bias, float(eps))
        ctx.save_for_backward(xc, weight, mean, rstd)
        ctx.groups, ctx.has_bias = int(groups), bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, rstd = ctx.saved_tensors
        dx, dg, db = _ext.load().group_norm_bwd(x, dy.float().contiguous(), weight, mean, rstd, ctx.groups)
        return dx, (dg if weight is not None else None), (db if ctx.has_bias else None), None, None


class _BatchNormNhwcFn(torch.autograd.Function):
    """Training-mode BatchNorm2d on a channels_last activation (csrc/misc.cu::bn_nhwc_*): 2 coalesced passes per direction, the
    running statistics are updated in place by the forward kernel."""

    @staticmethod
    def forward(ctx, x, weight, bias, run_mean, run_var, eps, momentum):
        xh = x.float().contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)       # NHWC view (free for channels_last)
        w = weight.detach().reshape(-1).contiguous() if weight is not None else None
        b = bias.detach().reshape(-1).contiguous() if bias is not None else None
        # the result is a fresh NCHW-logical channels_last tensor (NOT a view of a kernel output: ReLU(inplace=True) follows in
        # the torchvision blocks); the kernel writes through its NHWC view
        y = torch.empty_like(x, dtype=torch.float32, memory_format=torch.channels_last)
        mean, rstd = _ext.load().bn_nhwc_fwd(xh, y.permute(0, 2, 3, 1), w, b, run_mean, run_var, float(eps), float(momentum))
        ctx.save_for_backward(xh, w, mean, rstd)
        ctx.wshape = weight.shape if weight is not None else None
        ctx.has_bias = bias is not None
        ctx.bshape = bias.shape if bias is not None else None
        return y

    @staticmethod
    def backward(ctx, gy):
        xh, w, mean, rstd = ctx.saved_tensors
        g = gy.float().contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)
        dx, dw, db = _ext.load().bn_nhwc_bwd(xh, g, w, mean, rstd)
        return (dx.permute(0, 3, 1, 2), dw.view(ctx.wshape) if ctx.wshape is not None else None,
                db.view(ctx.bshape) if ctx.has_bias else None, None, None, None, None)


def batch_norm_train_nhwc(x, weight, bias, run_mean, run_var, eps: float, momentum: float):
    """Training-mode batch norm of a 4-D CUDA tensor through the NHWC kernels (weight / bias may be any shape with C elements)."""
    return _BatchNormNhwcFn.apply(x, weight, bias, run_mean, run_var, float(eps), float(momentum))


def group_norm(x, groups: int, weight=None, bias=None, eps: float = 1e-5):
    if native(x):
        if torch.is_grad_enabled() and (x.requires_grad or (weight is not None and weight.requires_grad)):
            return _GroupNormFn.apply(x, weight, bias, int(groups), float(eps))
        return _ext.load().group_norm_fwd(x.float().contiguous(), int(groups), weight, bias, float(eps))
    return ref.group_norm(x, groups, weight, bias, eps)
