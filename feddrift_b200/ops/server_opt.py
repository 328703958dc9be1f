"""FedOpt server step fused into the K1 aggregation epilogue (native path), and the per-slot server optimizer state of a
``ModelBank`` (``--server_optimizer`` of the continual engines)."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _ext

_KIND = {"sgd": 1, "adam": 2, "adagrad": 3, "yogi": 4}
B1, B2 = 0.9, 0.999


def native_server_opt_step_(theta, avg, state: Dict, opt: str, lr: float, momentum=0.0, b1=0.9, b2=0.999, eps=1e-8):
    """``theta`` [P] or [M,P] is stepped in place using the pseudo-gradient ``theta - avg``.
    Implemented by running the K1 kernel on a single 'client' (= avg) with the optimizer epilogue."""
    ext = _ext.load(required=True)
    th = theta.reshape(1, -1) if theta.dim() == 1 else theta
    M, P = th.shape
    cp = avg.reshape(1, M, P).contiguous()
    n = torch.ones(1, M, dtype=torch.float32, device=th.device)
    state["step"] = state.get("step", 0) + 1
    s0 = s1 = None
    if opt == "sgd":
        if momentum:
            s0 = state.setdefault("momentum", torch.zeros_like(th))
    elif opt == "adagrad":
        s0 = state.setdefault("sum", torch.zeros_like(th))
    else:
        s0 = state.setdefault("m", torch.zeros_like(th))
        s1 = state.setdefault("v", torch.full_like(th, 1e-6) if opt == "yogi" else torch.zeros_like(th))
    ext.cluster_aggregate_opt(th, cp, n, _KIND[opt], float(lr), float(momentum), float(b1), float(b2), float(eps),
                              int(state["step"]), s0, s1)
    return theta


class SlotServerOpt:
    """Server optimizer of every model slot of a ``ModelBank``: after slot m is averaged (total weight > 0), θ_m takes one
    ``opt`` step on the pseudo-gradient θ_m − avg_m (``reference.server_opt_step_`` law, β1 = 0.9, β2 = 0.999).

    Each slot owns its state rows (``s0``: sgd momentum buffer / Adagrad sum / first moment, ``s1``: second moment; both
    ``[M, P]``) and its step counter ``step [M]`` (Adam's bias correction), so a slot that does not aggregate in a round
    keeps its state and counter.  ``mask`` (bool ``[P]`` or None) marks the trainable entries: the others (BatchNorm
    running statistics, ``num_batches_tracked``) take the plain average and never enter the optimizer."""

    def __init__(self, opt: str, M: int, P: int, device, lr: float = 1.0, momentum: float = 0.0, eps: float = 1e-8,
                 mask: Optional[torch.Tensor] = None):
        if opt not in _KIND:
            raise ValueError(f"server optimizer must be one of none, {', '.join(_KIND)} (got {opt!r})")
        self.opt, self.kind = opt, _KIND[opt]
        self.lr, self.momentum, self.eps = float(lr), float(momentum), float(eps)
        z = lambda: torch.zeros(M, P, dtype=torch.float32, device=device)  # noqa: E731
        self.s0 = z() if (opt != "sgd" or self.momentum != 0.0) else None
        self.s1 = z() if opt in ("adam", "yogi") else None
        self.step = torch.zeros(M, dtype=torch.int32, device=device)
        self.mask = None if mask is None else mask.to(device=device, dtype=torch.bool)
        self._mask_u8 = None if mask is None else self.mask.to(torch.uint8).contiguous()
        self.reset()

    def reset(self, m: Optional[int] = None) -> None:
        """Initial state for slot ``m`` (all slots when None): zero moments and counter, Yogi's v₀ = 1e-6."""
        rows = slice(None) if m is None else m
        if self.s0 is not None:
            self.s0[rows] = 0.0
        if self.s1 is not None:
            self.s1[rows] = 1e-6 if self.opt == "yogi" else 0.0
        self.step[rows] = 0

    def tensors(self):
        return [t for t in (self.s0, self.s1, self.step) if t is not None]

    def aggregate_native_(self, theta, client_params, n) -> torch.Tensor:
        """K1 with the per-slot epilogue; returns the per-slot totals [M] and advances the counters of the slots with total > 0."""
        return _ext.load(required=True).cluster_aggregate_slots(
            theta, client_params.contiguous(), n.float().contiguous(), self.kind, self.lr, self.momentum, B1, B2, self.eps,
            self.s0, self.s1, self.step, self._mask_u8)

    def aggregate_reference_(self, theta, client_params, n) -> torch.Tensor:
        from . import reference as ref
        avg = theta.clone()
        tot = ref.cluster_aggregate_(avg, client_params, n)
        ref.server_opt_slots_(theta, avg, tot > 0, self.opt, self.s0, self.s1, self.step, self.lr, self.momentum, self.eps,
                              self.mask)
        return tot


def make_server_opt(args, M: int, P: int, device, weight_mask: Optional[torch.Tensor] = None) -> Optional[SlotServerOpt]:
    """``SlotServerOpt`` from ``args.server_optimizer`` / ``server_lr`` / ``server_momentum`` / ``server_eps``; None for
    ``none`` (plain FedAvg).  ``weight_mask`` is ``models.utils.weight_param_mask`` of the bank (None: all trainable)."""
    name = str(getattr(args, "server_optimizer", "none") or "none").lower()
    if name == "none":
        return None
    mask = None
    if weight_mask is not None and not bool(weight_mask[:P].all()):
        mask = weight_mask[:P]
    return SlotServerOpt(name, M, P, device, lr=float(getattr(args, "server_lr", 1.0)),
                         momentum=float(getattr(args, "server_momentum", 0.0)), eps=float(getattr(args, "server_eps", 1e-8)),
                         mask=mask)
