"""Flat parameter arena: every model slot is one fp32 row ``theta[m, :P]``.

This replaces the reference's per-model ``nn.Module`` + ``state_dict`` pickling
(``FedAvgEnsServerManager.py:25,66-67`` ships all M state_dicts to every rank every round;
``FedAvgEnsTrainerSoftCluster.py:51-58`` ``load_state_dict``s them).  With a row-per-model arena:

* ``state_dict(m)`` / ``load_state_dict(m, sd)`` are zero-copy views / one flat copy;
* aggregation, merge (FedDrift), clone-on-drift and re-initialisation are single fused kernels over
  rows (``ops.cluster_aggregate_``, ``ops.merge_axpby_``) instead of python ``for key`` loops;
* the same layout is what the multi-GPU symmetric-memory arena maps into every peer
  (``parallel/symm.py``): row m of GPU g is addressable from every GPU.

Rows are padded to a multiple of 32 floats (128 B) so rows start on cache-line / TMA-friendly boundaries.
"""
from __future__ import annotations

import copy
from typing import Dict, List, Optional

import torch
from torch import nn

from ..models import utils as mutils

ROW_ALIGN = 32  # floats


def padded(n: int, align: int = ROW_ALIGN) -> int:
    return (n + align - 1) // align * align


class ModelBank:
    """``num_models`` parameter rows sharing one architecture (the ``template`` module)."""

    _next_id = 0

    def __init__(self, template: nn.Module, num_models: int, device="cpu", storage: Optional[torch.Tensor] = None):
        self.template = copy.deepcopy(template).to("cpu")
        from ..ops.conv import convert_convs_
        convert_convs_(self.template)    # conv weights the rows store channels_last are consumed through TcConv2d (same state-dict keys)
        self.spec = mutils.flat_spec(self.template)
        self.P = mutils.flat_size(self.template)
        self.stride = padded(self.P)
        self.num_models = num_models
        self.device = torch.device(device)
        self.arena_id = ModelBank._next_id
        ModelBank._next_id += 1
        if storage is None:
            storage = torch.zeros(num_models, self.stride, dtype=torch.float32, device=self.device)
        assert storage.shape == (num_models, self.stride)
        self.storage = storage
        self.theta = storage[:, : self.P] if self.stride != self.P else storage
        self.mlp = self.template.mlp_spec() if hasattr(self.template, "mlp_spec") else None
        if self.mlp is not None and self.device.type == "cuda":
            # the register-resident MLP kernels are instantiated for the small drift-benchmark shapes only
            # (csrc/mlp.cuh FDB_MLP_SHAPES); bigger MLPs (fnn-MNIST 784→1568→10) take the nn.Module / TcLinear path
            from ..ops import small_round
            s_ = self.mlp
            if not small_round.supported(s_["kind"], s_["in"], s_["hidden"], s_["out"]):
                self.mlp = None
        # "every re-initialised model is identical" (reference reseeds before reset_parameters)
        mutils.reinitialize(self.template)
        self.init_row = mutils.flatten_state_dict(self.template.state_dict()).to(self.device)
        for m in range(num_models):
            self.theta[m].copy_(self.init_row)
        self._modules: Dict[int, nn.Module] = {}
        # per-slot server optimizer state (ops.server_opt.SlotServerOpt) or None: a slot that is re-initialised or
        # overwritten starts its optimizer afresh, so reinit / copy reset the destination slot's state here
        self.server_opt = None
        # the clients' error-feedback residual [C, M, P] of --compression eftopk or None: residual built up against a slot's
        # old model means nothing for its new one, so reinit / copy zero the destination slot's column for every client
        self.ef_res = None
        # the slots' centered-clipping state [M, P] of --aggregation_rule centered_clip (their previous outputs) or None: a
        # slot that is re-initialised or overwritten starts from a zero center, so reinit / copy zero its row
        self.cclip_center = None
        self.float_mask = torch.zeros(self.P, dtype=torch.bool)
        for _, _, dt, off, n in self.spec:
            self.float_mask[off:off + n] = bool(dt.is_floating_point)

    def rebind_storage(self, storage: torch.Tensor) -> None:
        """Move the bank onto ``storage`` ([num_models, ≥ P] fp32, e.g. the symmetric-memory θ buffer of the peer
        aggregation kernel): current values are copied once, afterwards rows written by the kernel ARE the bank — no
        per-round ``theta.copy_``.  Cached bank-bound modules are dropped (their parameters were views of the old rows)."""
        assert storage.shape[0] == self.num_models and storage.shape[1] >= self.P and storage.dtype == torch.float32
        storage[:, : self.P].copy_(self.theta)
        self.storage = storage
        self.stride = int(storage.stride(0))
        self.theta = storage[:, : self.P] if storage.shape[1] != self.P else storage
        self._modules = {}

    # -- state_dict interop ---------------------------------------------------------------
    def state_dict(self, m: int) -> "OrderedDict[str, torch.Tensor]":
        return mutils.unflatten_to_state_dict(self.theta[m], self.spec)

    def load_state_dict(self, m: int, sd) -> None:
        self.theta[m].copy_(mutils.flatten_state_dict(sd).to(self.device))

    def state_dicts(self) -> List["OrderedDict[str, torch.Tensor]"]:
        return [self.state_dict(m) for m in range(self.num_models)]

    # -- row ops --------------------------------------------------------------------------
    def copy(self, dst: int, src: int) -> None:
        if dst != src:
            self.theta[dst].copy_(self.theta[src])
            if self.server_opt is not None:
                self.server_opt.reset(dst)
            if self.ef_res is not None:
                self.ef_res[:, dst].zero_()
            if self.cclip_center is not None:
                self.cclip_center[dst].zero_()

    def reinit(self, m: int) -> None:
        self.theta[m].copy_(self.init_row)
        if self.server_opt is not None:
            self.server_opt.reset(m)
        if self.ef_res is not None:
            self.ef_res[:, m].zero_()
        if self.cclip_center is not None:
            self.cclip_center[m].zero_()

    def reset_parameters_random(self, m: int, generator: Optional[torch.Generator] = None) -> None:
        """Fresh (NOT reseeded) init — the IFCA 'hard' path at t=0 calls ``reset_parameters`` directly
        (``FedAvgEnsAggregatorSoftCluster.py:66-70``), giving each model different weights."""
        tmp = copy.deepcopy(self.template)
        if generator is not None:
            torch.manual_seed(int(torch.randint(0, 2 ** 31 - 1, (1,), generator=generator)))
        for layer in tmp.children():
            if hasattr(layer, "reset_parameters"):
                layer.reset_parameters()
        self.load_state_dict(m, tmp.state_dict())

    def merge(self, base: int, second: int, w1: float, w2: float) -> None:
        from .. import ops
        ops.merge_axpby_(self.theta, base, second, w1, w2)

    def to(self, device) -> "ModelBank":
        nb = ModelBank(self.template, self.num_models, device)
        nb.theta.copy_(self.theta.to(device))
        return nb

    def clone(self) -> "ModelBank":
        nb = ModelBank(self.template, self.num_models, self.device)
        nb.theta.copy_(self.theta)
        return nb

    # -- nn.Module bridge (big models / façade path) -----------------------------------
    def module(self, m: int) -> nn.Module:
        """An ``nn.Module`` whose parameters/buffers ARE views of row ``m`` (no copy, shares storage)."""
        mod = self._modules.get(m)
        if mod is None:
            mod = copy.deepcopy(self.template).to(self.device)
            views = self.state_dict(m)
            for name, p in list(mod.named_parameters()):
                _set_tensor(mod, name, nn.Parameter(views[name], requires_grad=p.requires_grad))
            for name, b in list(mod.named_buffers()):
                if name in views and views[name].dtype == b.dtype:
                    _set_tensor(mod, name, views[name], buffer=True)
            self._modules[m] = mod
        return mod

    def forward(self, m: int, x: torch.Tensor, train: bool = False) -> torch.Tensor:
        if self.mlp is not None:
            from ..ops import mlp_forward
            s = self.mlp
            return mlp_forward(self.theta[m], x.reshape(x.shape[0], -1), s["kind"], s["in"], s["hidden"], s["out"])
        mod = self.module(m)
        mod.train(train)
        return mod(x)


def _set_tensor(mod: nn.Module, dotted: str, value, buffer: bool = False) -> None:
    parts = dotted.split(".")
    for p in parts[:-1]:
        mod = getattr(mod, p)
    if buffer:
        mod._buffers[parts[-1]] = value
    else:
        mod._parameters[parts[-1]] = value


class ClientArena:
    """Per-(client, model) training state: local params + Adam(amsgrad) moments, all flat rows.

    Layout ``[C, M, P]`` so that the K1 aggregation kernel reads ``client_params[:, m, :]`` with a fixed
    stride and the fused optimizer kernel walks contiguous rows.  Optimizer state persists across rounds
    inside a time step and is reset between time steps (the reference gets this implicitly from
    relaunching the process per time step — ``FedAvgEnsTrainer.py:25-33``, SURVEY §7.3)."""

    def __init__(self, num_clients: int, num_models: int, P: int, device="cpu", adam: bool = True, ef: bool = False):
        self.C, self.M, self.P = num_clients, num_models, P
        self.device = torch.device(device)
        z = lambda: torch.zeros(num_clients, num_models, P, dtype=torch.float32, device=self.device)  # noqa: E731
        self.params = z()
        self.m = z() if adam else None
        self.v = z() if adam else None
        self.vmax = z() if adam else None
        self.step = torch.zeros(num_clients, num_models, dtype=torch.int32, device=self.device)
        self.n = torch.zeros(num_clients, num_models, dtype=torch.float32, device=self.device)
        # error-feedback residual of --compression eftopk (the part of each (client, slot) update not uploaded yet)
        self.ef_res = z() if ef else None

    def reset_optimizer(self) -> None:
        """Start of a time step: the client optimizer state and the error-feedback residual start from zero."""
        for t in (self.m, self.v, self.vmax, self.ef_res):
            if t is not None:
                t.zero_()
        self.step.zero_()
