"""FedML-compatible ``fedavg_ens`` package: the message-driven continual trainer with drift algorithms.

API parity with ``fedml_api/distributed/fedavg_ens/`` (SURVEY §2.2): ``FedML_init``,
``FedML_FedAvgEns_data_loader``, ``FedML_FedAvgEns_distributed``, ``MyMessage``, ``FedAvgEnsServerManager``,
``FedAvgEnsClientManager``, the ``FedAvgEnsAggregator*`` family and the ``FedAvgEnsTrainer*`` family — same
constructor/handler surface, same wire protocol (SURVEY Appendix C), so a reference experiment script ports by
changing imports.  This is the rank-per-process / in-process *façade* path (gloo or INPROC transports); the
device engine (``sim.DriftSim``) is the fast path and shares every state machine with it.

Differences by design (documented, SURVEY §7.3):
* server-side models live in a :class:`ModelBank` (flat rows); uploads land in a ``[C, M, P]`` arena and the
  per-model weighted average is ONE ``ops.cluster_aggregate_`` call instead of python ``for key: for client:``;
* ``model_params`` may travel as a :class:`DeviceRef` (zero-copy) on the INPROC/STREAM transports;
* drift state is held by a :class:`StateStore` (memory or a directory) instead of pickles in CWD;
* ``finish`` stops the managers cooperatively; the time-step loop runs in-process (no ``mpirun`` per time step).
"""
from __future__ import annotations

import copy
import logging
import os
import pickle
from typing import Dict, Optional

import numpy as np
import torch
from torch import nn

from .. import ops
from ..core.comm.inproc import World
from ..core.managers import RoundWatchdog, ClientManager, ServerManager
from ..core.message import DeviceRef, Message
from ..data import changepoints as cpmod
from ..data.drift import DEFAULT_DELTAS, DriftData
from ..models import utils as mutils
from ..core.robustness import make_defense
from ..ops.reference import (aggregation_params, attack_params, attack_seed, attacker_clients, cclip_params, compress_seed,
                             compression_params, geomed_params, krum_params, prox_mu_param, topk_k, topk_ratio_param)
from ..ops.server_opt import make_server_opt
from ..parallel.arena import ModelBank
from ..utils.metrics import get_sink
from .evaluator import Evaluator
from .softcluster import SoftClusterState
from .states import AdaState, DriftSurfState, KueState, MultiModelAccState, aue_model_num

ARENAS: Dict[int, ModelBank] = {}


class MyMessage:
    """Message type / payload-key constants (parity: ``message_define.py:1-23``)."""
    MSG_TYPE_S2C_INIT_CONFIG = 1
    MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT = 2
    MSG_TYPE_C2S_SEND_MODEL_TO_SERVER = 3
    MSG_TYPE_C2S_SEND_STATS_TO_SERVER = 4
    MSG_ARG_KEY_TYPE = "msg_type"
    MSG_ARG_KEY_SENDER = "sender"
    MSG_ARG_KEY_RECEIVER = "receiver"
    MSG_ARG_KEY_MODEL_PARAMS = "model_params"
    MSG_ARG_KEY_CLIENT_INDEX = "client_idx"
    MSG_ARG_KEY_MODEL_AND_NUM_SAMPLES = "model_and_num_samples"
    MSG_ARG_KEY_EXTRA_INFO = "extra_info"


class StateStore:
    """Drift-state persistence across time steps (replaces sc_state.pkl / mm_state.pkl / ds_state.pkl /
    ada_state.pkl / kue_state.pkl / model_params.pt in CWD).  ``path=None`` keeps everything in memory."""

    def __init__(self, path: Optional[str] = None):
        self.path, self.mem = path, {}
        if path:
            os.makedirs(path, exist_ok=True)

    def put(self, key: str, obj) -> None:
        self.mem[key] = obj
        if self.path:
            tmp = os.path.join(self.path, key + ".tmp")
            with open(tmp, "wb") as fh:
                pickle.dump(obj, fh)
            os.replace(tmp, os.path.join(self.path, key + ".pkl"))

    def get(self, key: str, default=None):
        if key in self.mem:
            return self.mem[key]
        if self.path and os.path.exists(os.path.join(self.path, key + ".pkl")):
            with open(os.path.join(self.path, key + ".pkl"), "rb") as fh:
                self.mem[key] = pickle.load(fh)
            return self.mem[key]
        return default

    def clear(self) -> None:
        self.mem.clear()
        if self.path:
            for f in os.listdir(self.path):
                if f.endswith(".pkl"):
                    os.remove(os.path.join(self.path, f))


class _Comm:
    """What ``FedML_init`` returns as ``comm``: carries the transport handle + a Barrier (MPI-like surface)."""

    def __init__(self, backend: str, world=None, rank: int = 0, size: int = 1, device: str = "cpu"):
        self.backend, self.world, self.rank, self.size, self.device = backend, world, rank, size, device
        self.group = None

    def Barrier(self) -> None:
        if self.backend in ("GLOO", "NCCL", "MPI", "DIST"):
            import torch.distributed as dist
            if dist.is_initialized():
                dist.barrier()

    def Get_rank(self) -> int:
        return self.rank

    def Get_size(self) -> int:
        return self.size


def FedML_init(backend: str = "GLOO", world_size: Optional[int] = None):
    """-> (comm, process_id, worker_number).  ``GLOO``/``NCCL``: reads RANK/WORLD_SIZE/MASTER_* (torchrun);
    ``INPROC``: one process hosts ``world_size`` logical ranks (parity: ``FedAvgEnsAPI.py:25-29``)."""
    backend = backend.upper()
    if backend in ("INPROC", "STREAM"):
        size = int(world_size or 1)
        return _Comm(backend, World(size), 0, size), 0, size
    import torch.distributed as dist
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        dist.init_process_group("nccl" if backend == "NCCL" else "gloo")
    return _Comm("DIST", None, dist.get_rank(), dist.get_world_size(),
                 "cuda" if backend == "NCCL" else "cpu"), dist.get_rank(), dist.get_world_size()


def FedML_finalize() -> None:
    """Orderly end of a distributed run (the reference ends with ``MPI.COMM_WORLD.Abort()``)."""
    import torch.distributed as dist
    if dist.is_initialized():
        from ..core.comm.dist import shutdown_transport
        shutdown_transport()


# ====================================================================================== data loaders
def _with(args, **kw):
    a = copy.copy(args)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def FedML_FedAvgEns_data_loader(args, loader_func, device, comm, process_id, store: Optional[StateStore] = None,
                                bank: Optional[ModelBank] = None, evaluator: Optional[Evaluator] = None):
    """Per-algorithm list of datasets (one FedML tuple per model slot) — dispatch parity with
    ``FedAvgEnsAPI.py:31-60``.  ``loader_func(args)`` must honour ``args.retrain_data``."""
    store = store if store is not None else getattr(args, "state_store", None) or _default_store()
    algo, t = args.concept_drift_algo, args.curr_train_iteration

    def load(retrain):
        return loader_func(_with(args, retrain_data=retrain))

    if algo in ("aue", "auepc"):
        return [load(f"win-{m + 1}") for m in range(aue_model_num(t, args.ensemble_window))]
    if algo == "kue":
        ds = [load("poisson") for _ in range(args.concept_num)]
        if t == 0 and process_id == 0:
            store.put("kue_state", KueState(args.concept_num, ds[0][-1], np.random.RandomState(args.dummy_arg)))
        comm.Barrier()
        return ds
    if algo == "ada":
        if t == 0 and process_id == 0:
            store.put("ada_state", AdaState(init_lr=args.lr))
        comm.Barrier()
        return [load(args.concept_drift_algo_arg.split("_")[0])]
    if algo in ("exp", "lin"):
        return [load("win-1")]
    if algo == "driftsurf":
        if t == 0:
            d = 0.01 * float(args.concept_drift_algo_arg or 0) or {"sea": 0.02, "sine": 0.10, "circle": 0.05}.get(args.dataset, 0.05)
            st = DriftSurfState(delta=d)
            ds = [load("sel-0"), load("sel-0")]
        else:
            st = store.get("ds_state")
            if process_id == 0 and bank is not None and evaluator is not None:
                st.run_ds_algo(bank, evaluator, t, scratch_row=bank.num_models - 1)
            ds = [load("sel-" + ",".join(str(x) for x in st.get_train_data(k))) for k in st.get_train_keys()]
        if process_id == 0:
            store.put("ds_state", st)
        comm.Barrier()
        return ds
    if algo in ("mmacc", "mmgeni", "mmgeniex"):
        if t == 0:
            st = MultiModelAccState(args.client_num_in_total, args.concept_num, DEFAULT_DELTAS.get(args.dataset, 0.1))
        else:
            st = store.get("mm_state")
        if algo == "mmacc":
            st.run_model_select(evaluator if t > 0 else None, t)
        else:
            cps = cpmod.load(args.change_points, args.total_train_iteration, args.client_num_in_total,
                             bool(args.drift_together), args.time_stretch)
            (st.model_select_geni if algo == "mmgeni" else st.model_select_geniex)(t, cps, args.time_stretch)
        ds = []
        for m in range(args.concept_num):
            td = st.get_train_data_by_model(m)
            if td != "":
                st.set_model(m)
                ds.append(load("clientsel-" + td))
        if process_id == 0:
            store.put("mm_state", st)
        comm.Barrier()
        return ds
    if algo == "clusterfl":
        return [load(args.concept_drift_algo_arg) for _ in range(args.concept_num)]
    if algo in ("softcluster", "softclusterwin-1", "softclusterreset"):
        if t == 0 and process_id == 0:
            cps = None
            if args.concept_drift_algo_arg == "geni":
                cps = cpmod.load(args.change_points, args.total_train_iteration, args.client_num_in_total,
                                 bool(args.drift_together), args.time_stretch)
            store.put("sc_state", SoftClusterState.from_args(args, cps, rng=np.random.RandomState(args.dummy_arg),
                                                             max_steps=args.total_train_iteration + 2))
        comm.Barrier()
        one = load("win-1")
        return [one for _ in range(args.concept_num)]  # M = concept_num slots always allocated
    raise NameError("concept_drift_algo")


_STORE: Optional[StateStore] = None


def _default_store() -> StateStore:
    global _STORE
    if _STORE is None:
        _STORE = StateStore(None)
    return _STORE


# ====================================================================================== trainers (clients)
class FedAvgEnsTrainer:
    """Base client trainer (aue / auepc / driftsurf / mm*): ``epochs`` single-minibatch steps per model, Adam
    (amsgrad, wd) by default, optimizer state kept across rounds (parity: ``FedAvgEnsTrainer.py:10-95``)."""

    def __init__(self, client_index, train_data_local_dicts, train_data_local_num_dicts, train_data_nums,
                 all_local_data, device, models, args):
        self.client_index = client_index
        self.train_data_local_dicts = train_data_local_dicts
        self.train_data_local_num_dicts = train_data_local_num_dicts
        self.all_train_data_nums = train_data_nums
        self.all_local_data = all_local_data
        self.device, self.args, self.models = device, args, models
        self.extra_info = None
        self.criterions = [nn.CrossEntropyLoss().to(device) for _ in models]
        self.optimizers = [self._make_optimizer(m) for m in models]
        self.rng = np.random.RandomState(int(getattr(args, "dummy_arg", 0)) * 1000 + int(client_index) + 1)
        self.fedprox_mu = prox_mu_param(getattr(args, "fedprox_mu", 0.0))

    def _make_optimizer(self, m):
        if self.args.client_optimizer == "sgd":
            return torch.optim.SGD(m.parameters(), lr=self.args.lr)
        return torch.optim.Adam(filter(lambda p: p.requires_grad, m.parameters()), lr=self.args.lr,
                                weight_decay=self.args.wd, amsgrad=True)

    def update_model(self, weights, extra_info):
        if isinstance(weights, DeviceRef):  # zero-copy: read the server arena rows in place
            bank = ARENAS[weights.arena_id]
            weights = [bank.state_dict(r) for r in weights.rows]
        for m, w in zip(self.models, weights):
            if getattr(self.args, "is_mobile", 0) == 1:
                w = {k: torch.as_tensor(v) for k, v in w.items()}
            m.load_state_dict(w)
        self.extra_info = extra_info

    def update_dataset(self, client_index):
        self.client_index = client_index

    # -- hooks ----------------------------------------------------------------------------
    def _plan(self, mod_idx):
        """-> (local_sample_number, sampler() -> (x, y)) or (0, None) to skip."""
        n = self.train_data_local_num_dicts[mod_idx].get(self.client_index, 0)
        if n == 0:
            return 0, None
        batches = self.train_data_local_dicts[mod_idx][self.client_index]
        if isinstance(batches, list):
            return n, lambda: batches[self.rng.choice(len(batches))]
        return n, lambda: next(iter(batches))

    def _transform(self, mod_idx, x):
        return x

    def _before_train(self, mod_idx):
        ...

    def train(self):
        results = {}
        for mod_idx, model in enumerate(self.models):
            n, sampler = self._plan(mod_idx)
            if n == 0 or sampler is None:
                results[mod_idx] = (None, 0)
                continue
            model.to(self.device)
            model.train()
            self._before_train(mod_idx)
            opt, crit = self.optimizers[mod_idx], self.criterions[mod_idx]
            # FedProx (--fedprox_mu): the local objective gains mu/2‖w − w0‖² over the trainable parameters, w0 = the received model
            prox = [(p, p.detach().clone()) for p in model.parameters() if p.requires_grad] if self.fedprox_mu > 0 else []
            for _ in range(self.args.epochs):
                x, labels = sampler()
                x, labels = self._transform(mod_idx, x.to(self.device)), labels.to(self.device)
                opt.zero_grad()
                loss = crit(model(x), labels)
                loss.backward()
                for p, p0 in prox:
                    if p.grad is not None:
                        p.grad.add_(p.detach() - p0, alpha=self.fedprox_mu)
                opt.step()
            weights = {k: v.detach().cpu() for k, v in model.state_dict().items()}
            if getattr(self.args, "is_mobile", 0) == 1:
                weights = {k: v.tolist() for k, v in weights.items()}
            results[mod_idx] = (weights, n)
        return results


class FedAvgEnsTrainerSoftCluster(FedAvgEnsTrainer):
    """Data selection from ``extra_info['sc_weights'][t][m][c]`` over all past time steps
    (parity: ``FedAvgEnsTrainerSoftCluster.py:63-135``)."""

    def _plan(self, mod_idx):
        w = self.extra_info["sc_weights"]
        t_cur = self.args.curr_train_iteration
        if not np.any(w[t_cur][mod_idx]):
            return 0, None
        T = len(self.all_local_data)
        unnorm = np.asarray([w[t][mod_idx][self.client_index] * len(self.all_local_data[t]) if t in w else 0.0
                             for t in range(T)])
        n = float(unnorm.sum())
        if n == 0:
            return 0, None
        if all(isinstance(self.all_local_data[t], list) for t in range(T)):
            pool = [b for t in range(T) if unnorm[t] > 0 for b in self.all_local_data[t]]
            return n, lambda: pool[self.rng.choice(len(pool))]
        probs = unnorm / n
        return n, lambda: next(iter(self.all_local_data[self.rng.choice(T, p=probs)]))


class _TimeWeightedTrainer(FedAvgEnsTrainer):
    def _weights(self, T):
        raise NotImplementedError

    def _plan(self, mod_idx):
        T = len(self.all_local_data)
        n = sum(len(self.all_local_data[t]) for t in range(T))
        if n == 0:
            return 0, None
        probs = self._weights(T)
        probs = probs / probs.sum()

        def sampler():
            data_t = self.all_local_data[self.rng.choice(T, p=probs)]
            return data_t[self.rng.choice(len(data_t))] if isinstance(data_t, list) else next(iter(data_t))
        return n, sampler


class FedAvgEnsTrainerExp(_TimeWeightedTrainer):
    def _weights(self, T):
        return np.asarray([2.0 ** t for t in range(T)])


class FedAvgEnsTrainerLin(_TimeWeightedTrainer):
    def _weights(self, T):
        return np.asarray([t + 1.0 for t in range(T)])


class FedAvgEnsTrainerAda(FedAvgEnsTrainer):
    def _make_optimizer(self, m):  # forced SGD (FedAvgEnsTrainerAda.py:28-30)
        return torch.optim.SGD(m.parameters(), lr=self.args.lr)

    def _before_train(self, mod_idx):
        for g in self.optimizers[mod_idx].param_groups:
            g["lr"] = self.extra_info["lr"]


class FedAvgEnsTrainerKue(FedAvgEnsTrainer):
    def _transform(self, mod_idx, x):
        mask = torch.as_tensor(np.asarray(self.extra_info["masks"][mod_idx]), dtype=x.dtype, device=x.device)
        return x * mask.reshape((1,) + tuple(x.shape[1:]))


class FedAvgEnsTrainerClusterFL(FedAvgEnsTrainer):
    def _plan(self, mod_idx):
        if int(self.extra_info[self.client_index]) != mod_idx:
            return 0, None
        return super()._plan(mod_idx)


# ====================================================================================== aggregators (server)
class _BaseAggregator:
    """Bookkeeping + K1 aggregation shared by every ``FedAvgEnsAggregator*``."""

    defend_uploads = True   # apply ``--defense_type`` in ``_aggregate_models`` (single-model FedAvg defends in its own hook)

    def __init__(self, train_globals, test_globals, all_train_data_nums, train_data_local_dicts, test_data_local_dicts,
                 train_data_local_num_dicts, all_data, worker_num, device, models, class_num, args):
        self.train_globals, self.test_globals = train_globals, test_globals
        self.all_train_data_nums, self.all_data = all_train_data_nums, all_data
        self.train_data_local_dicts, self.test_data_local_dicts = train_data_local_dicts, test_data_local_dicts
        self.train_data_local_num_dicts = train_data_local_num_dicts
        self.worker_num, self.device, self.class_num, self.args = worker_num, torch.device(device), class_num, args
        self.sink = get_sink()
        self.store: StateStore = getattr(args, "state_store", None) or _default_store()
        if isinstance(models, ModelBank):
            self.bank = models
        else:
            self.bank = ModelBank(models[0], len(models), self.device)
            for i, m in enumerate(models):
                self.bank.load_state_dict(i, m.state_dict())
        ARENAS[self.bank.arena_id] = self.bank
        # per-slot server optimizer (--server_optimizer): fresh state for every aggregator, i.e. every time step
        wmask = mutils.weight_param_mask(self.bank.spec)[: self.bank.P]
        self.bank.server_opt = make_server_opt(args, self.bank.num_models, self.bank.P, self.device, wmask)
        # robust aggregation (--defense_type) of the uploads; its noise round counts this aggregator's aggregations
        self.defense = make_defense(args) if self.defend_uploads else None
        self.defense_mask = None if bool(wmask.all()) else wmask.to(self.device)
        self._defense_round = 0
        # cluster aggregation rule (--aggregation_rule / --trim_ratio): None is the weighted mean, (rule, β) the coordinate-wise
        # median / trimmed mean over the workers that uploaded a model for the slot (each counted once)
        rule, beta = aggregation_params(getattr(args, "aggregation_rule", "mean") or "mean", getattr(args, "trim_ratio", 0.1))
        # the geometric median (--geomed_iters / --geomed_nu, validated whatever the rule) carries (rule, β, R, ν); its
        # distances cover the trainable entries (defense_mask)
        gm_iters, gm_nu = geomed_params(getattr(args, "geomed_iters", 4), getattr(args, "geomed_nu", 1e-6))
        # Multi-Krum (--krum_f / --krum_m, validated whatever the rule) carries (rule, β, f, m), distances as above
        krum_f, krum_m = krum_params(getattr(args, "krum_f", 1), getattr(args, "krum_m", 1))
        # centered clipping (--cclip_tau / --cclip_iters, validated whatever the rule) carries (rule, β, τ, L), distances as
        # above; the aggregator is rebuilt every time step, so the bank's per-slot centers start at zero here
        cc_tau, cc_iters = cclip_params(getattr(args, "cclip_tau", 1.0), getattr(args, "cclip_iters", 1))
        self.bank.cclip_center = None
        if rule == "mean":
            self.agg_rule = None
        elif rule == "geometric_median":
            self.agg_rule = (rule, beta, gm_iters, gm_nu)
        elif rule == "multi_krum":
            self.agg_rule = (rule, beta, krum_f, krum_m)
        elif rule == "centered_clip":
            self.agg_rule = (rule, beta, cc_tau, cc_iters)
            self.bank.cclip_center = torch.zeros(self.bank.num_models, self.bank.P, dtype=torch.float32, device=self.device)
        else:
            self.agg_rule = (rule, beta)
        # upload compression (--compression qsgd): each arriving upload is quantized against bank.theta[m]; its draws follow
        # this aggregator's round counter, advanced when a round's uploads are complete (packages without the flags: none)
        self.q_level, self.q_bucket = compression_params(getattr(args, "compression", "none") or "none",
                                                         getattr(args, "quantize_level", 16), getattr(args, "quantize_bucket", 512))
        self._compress_round = 0
        self.models = [self.bank.module(i) for i in range(self.bank.num_models)]
        M, P = self.bank.num_models, self.bank.P
        # top-k with error feedback (--compression eftopk): each arriving upload is sparsified against bank.theta[m] with the
        # residual of the CLIENT the worker trained this round (client_sampling's list), not of the worker row; the
        # aggregator is rebuilt every time step, so the residual starts at zero there
        self.topk_ratio = topk_ratio_param(getattr(args, "topk_ratio", 0.01))
        self.topk_k = topk_k(self.topk_ratio, int(wmask.sum())) \
            if (getattr(args, "compression", "none") or "none") == "eftopk" else 0
        n_clients = int(getattr(args, "client_num_in_total", worker_num) or worker_num)
        self.ef_res = torch.zeros(max(n_clients, worker_num), M, P, dtype=torch.float32, device=self.device) \
            if self.topk_k else None
        self.bank.ef_res = self.ef_res
        self._round_clients = None
        # simulated Byzantine clients (--attack_type / --attack_clients / --attack_scale, validated whatever the type): the
        # run's attacker set over CLIENTS; a round's uploads are poisoned once all of them have arrived (the attacker model
        # sits at the aggregator, as in later FedML releases), rows mapped to clients through client_sampling's list
        atk, atk_a, atk_s = attack_params(getattr(args, "attack_type", "none") or "none", getattr(args, "attack_clients", 0),
                                          getattr(args, "attack_scale", 1.0), n_clients)
        self.attackers = attacker_clients(n_clients, atk_a, int(getattr(args, "dummy_arg", 0)))
        self.attack = (atk, atk_s) if atk != "none" and atk_a > 0 else None
        self.upload = torch.zeros(worker_num, M, P, dtype=torch.float32, device=self.device)
        self.upload_n = torch.zeros(worker_num, M, dtype=torch.float32, device=self.device)
        self.flag_client_model_uploaded_dict = {i: False for i in range(worker_num)}
        self.weights_and_num_samples_dict: Dict[int, Dict] = {}

    # -- FedML surface ------------------------------------------------------------------
    def get_global_model_params(self):
        if getattr(self.args, "zero_copy", 0):
            return DeviceRef(self.bank.arena_id, range(self.bank.num_models))
        return [{k: v.detach().cpu().clone() for k, v in self.bank.state_dict(m).items()}
                for m in range(self.bank.num_models)]

    def add_local_trained_result(self, index, weights_and_num_samples):
        self.weights_and_num_samples_dict[index] = weights_and_num_samples
        for m, (sd, n) in weights_and_num_samples.items():
            m = int(m)
            self.upload_n[index, m] = float(n) if sd is not None else 0.0
            if sd is not None and n > 0:
                if getattr(self.args, "is_mobile", 0) == 1:
                    sd = {k: torch.as_tensor(v) for k, v in sd.items()}
                self.upload[index, m].copy_(mutils.flatten_state_dict(sd).to(self.device))
        if self.q_level:   # the client quantized before it uploaded: row = worker index · M + m
            sel = torch.zeros(self.worker_num, self.bank.num_models, dtype=torch.float32)
            for m, (sd, n) in weights_and_num_samples.items():
                if sd is not None and n > 0:
                    sel[index, int(m)] = 1.0
            if bool(sel.any()):
                a = self.args
                seed = int(getattr(a, "dummy_arg", 0)) * 7919 + 13 + 1000003 * int(getattr(a, "curr_train_iteration", 0) or 0)
                ops.qsgd_slots_(self.upload, self.bank.theta, sel.to(self.device), self.q_level, self.q_bucket, self.defense_mask,
                                compress_seed(seed, self._compress_round))
        if self.topk_k:   # the client sparsified before it uploaded, with its own residual
            sel = torch.zeros(1, self.bank.num_models, dtype=torch.float32)
            for m, (sd, n) in weights_and_num_samples.items():
                if sd is not None and n > 0:
                    sel[0, int(m)] = 1.0
            if bool(sel.any()):
                c = int(self._round_clients[index]) if self._round_clients is not None else int(index)
                ops.eftopk_slots_(self.upload[index:index + 1], self.bank.theta, self.ef_res[c:c + 1], sel.to(self.device),
                                  self.topk_k, self.defense_mask)
        self.flag_client_model_uploaded_dict[index] = True

    def check_whether_all_receive(self):
        if not all(self.flag_client_model_uploaded_dict[i] for i in range(self.worker_num)):
            return False
        for i in range(self.worker_num):
            self.flag_client_model_uploaded_dict[i] = False
        if self.attack is not None:
            self._attack_uploads()
        self._compress_round += 1
        return True

    def _attack_uploads(self):
        """Poison the complete round's upload arena in place (``ops.attack_slots_``) before any consumer reads it: row w is
        worker w, which trained client ``_round_clients[w]`` this round; the noise follows the round counter."""
        W = self.worker_num
        clients = self._round_clients if self._round_clients is not None else range(W)
        rows = torch.tensor([bool(self.attackers[int(c)]) for c in list(clients)[:W]], dtype=torch.bool)
        a = self.args
        seed = int(getattr(a, "dummy_arg", 0)) * 7919 + 13 + 1000003 * int(getattr(a, "curr_train_iteration", 0) or 0)
        ops.attack_slots_(self.upload, self.bank.theta, self.upload_n, rows, self.attack[0], self.attack[1], self.defense_mask,
                          attack_seed(seed, self._compress_round))

    def _aggregate_models(self, model_mask: Optional[np.ndarray] = None):
        n = self.upload_n.clone()
        if model_mask is not None:
            n[:, ~torch.as_tensor(model_mask, dtype=torch.bool, device=n.device)] = 0.0
        if self.defense is not None:   # row = worker index · M + m; the engine's seed of this time step
            self._defense_round += 1
            a = self.args
            seed = int(getattr(a, "dummy_arg", 0)) * 7919 + 13 + 1000003 * int(getattr(a, "curr_train_iteration", 0) or 0)
            self.defense.defend_slots_(self.upload, self.bank.theta, n, self.defense_mask, seed, self._defense_round)
        if self.agg_rule is not None and self.agg_rule[0] == "centered_clip":
            ops.cluster_aggregate_(self.bank.theta, self.upload, n, self.bank.server_opt, self.agg_rule, mask=self.defense_mask,
                                   center=self.bank.cclip_center)
        elif self.agg_rule is not None and self.agg_rule[0] in ("geometric_median", "multi_krum"):
            ops.cluster_aggregate_(self.bank.theta, self.upload, n, self.bank.server_opt, self.agg_rule, mask=self.defense_mask)
        else:
            ops.cluster_aggregate_(self.bank.theta, self.upload, n, self.bank.server_opt, self.agg_rule)

    def aggregate(self, round_idx):
        self._aggregate_models()
        return self.get_global_model_params()

    def client_sampling(self, round_idx, client_num_in_total, client_num_per_round):
        if client_num_in_total == client_num_per_round:
            return list(range(client_num_in_total))
        np.random.seed(round_idx)  # same clients per round across runs (reference behaviour)
        return np.random.choice(range(client_num_in_total), min(client_num_per_round, client_num_in_total), replace=False)

    def sample_round_clients(self, round_idx, client_num_in_total, client_num_per_round):
        """``client_sampling``, remembered: worker w trains entry w of the list in round ``round_idx``, so the round's
        uploads find their clients' error-feedback residuals."""
        idx = self.client_sampling(round_idx, client_num_in_total, client_num_per_round)
        self._round_clients = idx
        return idx

    def extra_info(self, round_idx):
        return None

    def reported_acc(self, correct, num_sample):
        return -1 if num_sample == 0 else correct / num_sample

    # -- evaluation ---------------------------------------------------------------------
    def _infer(self, model_idx, test_data, mask=None):
        """(correct, total, loss_sum) of model ``model_idx`` on a list of (x, y) batches — device-accumulated."""
        acc = torch.zeros(3, dtype=torch.float32, device=self.device)
        if test_data is None:
            return 0.0, 0.0, 0.0
        with torch.no_grad():
            for x, y in test_data:
                x = x.to(self.device)
                if mask is not None:
                    x = x * mask
                ops.eval_logits(self.bank.forward(model_idx, x), y.to(self.device), acc)
        a = acc.tolist()
        return a[0], a[2], a[1]

    def _route(self, client_idx):
        """-> (train_model, train_data, test_model, test_data) for the per-round evaluation."""
        raise NotImplementedError

    def _test_client(self, client_idx):
        mtr, dtr, mte, dte = self._route(client_idx)
        tr = self._infer(mtr, dtr)
        te = self._infer(mte, dte)
        return tr, te

    def test_on_all_clients(self, round_idx):
        a = self.args
        if round_idx % a.frequency_of_the_test == 0 or round_idx == a.comm_round - 1:
            tr_c = tr_n = tr_l = te_c = te_n = te_l = 0.0
            for c in range(a.client_num_in_total):
                (k, n, l), (k2, n2, l2) = self._test_client(c)
                tr_c, tr_n, tr_l, te_c, te_n, te_l = tr_c + k, tr_n + n, tr_l + l, te_c + k2, te_n + n2, te_l + l2
                if a.report_client == 1:
                    self.sink.log({f"Train/Acc-CL-{c}": self.reported_acc(k, n), "round": round_idx})
                    self.sink.log({f"Test/Acc-CL-{c}": self.reported_acc(k2, n2), "round": round_idx})
                self._after_client_eval(c, k, n)
                if getattr(a, "ci", 0) == 1:
                    break
            self.sink.log({"Train/Acc": tr_c / max(tr_n, 1), "round": round_idx})
            self.sink.log({"Train/Loss": tr_l / max(tr_n, 1), "round": round_idx})
            self.sink.log({"Test/Acc": te_c / max(te_n, 1), "round": round_idx})
            if self._report_test_loss:
                self.sink.log({"Test/Loss": te_l / max(te_n, 1), "round": round_idx})
            logging.info({"training_acc": tr_c / max(tr_n, 1), "test_acc": te_c / max(te_n, 1)})
        if round_idx > (a.comm_round - 5):
            self._save_state()

    _report_test_loss = True

    def _after_client_eval(self, c, correct, n):
        ...

    def _save_state(self):
        ...


class FedAvgEnsAggregatorSoftCluster(_BaseAggregator):
    """FedDrift server (parity: ``FedAvgEnsAggregatorSoftCluster.py:16-355``)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.data: Optional[DriftData] = getattr(self.args, "drift_data", None)
        self.evaluator = Evaluator(self.bank, self.data.to(self.device) if self.data is not None else None,
                                   self.args.batch_size) if self.data is not None else _ListEvaluator(self)
        self.sc_state: SoftClusterState = self.init_sc_state()

    def init_sc_state(self):
        a, st = self.args, self.store.get("sc_state")
        st._sink = self.sink
        t, arg, bank, ev = a.curr_train_iteration, a.concept_drift_algo_arg, self.bank, self.evaluator
        if "H" in arg:
            st.cluster_init() if t == 0 else st.cluster_hierarchical(t, bank, ev)
        elif "cfl" in arg:
            st.cluster_init() if t == 0 else st.cluster_cfl_init(t)
        elif "hard" in arg:
            if t == 0:
                g = torch.Generator().manual_seed(int(a.dummy_arg) + 12345)
                for m in range(bank.num_models):
                    bank.reset_parameters_random(m, g)
            st.cluster(ev.acc_matrix(list(range(bank.num_models)), t), t, 0)
        elif "mmacc" in arg:
            st.cluster_init() if t == 0 else st.cluster_mmacc2(t, bank, ev)
        else:
            if t == 0:
                st.cluster_init()
            else:
                acc = ev.acc_matrix(list(range(bank.num_models)), t)
                if a.concept_drift_algo == "softclusterreset":
                    deleted = []
                    for m in reversed(range(bank.num_models)):
                        rest = np.delete(acc, deleted + [m], axis=0)
                        if rest.shape[0] > 0 and np.all(acc[m] < np.max(rest, axis=0) + 0.01):
                            deleted.append(m)
                            self.sink.set_summary(f"Reset-{m}", 1)
                            st.set_weights_zero_model(m)
                            bank.reinit(m)
                    if deleted:
                        acc = ev.acc_matrix(list(range(bank.num_models)), t)
                st.cluster(acc, t, 0)
        if a.concept_drift_algo == "softclusterwin-1":
            st.set_weights_win1(t)
        if t == 0:
            for c in range(a.client_num_in_total):
                k, n, _ = self._infer(st.get_test_model_idx(0, c), self.all_data[c][0])
                st.set_acc(c, k / n if n else 0)
        return st

    def aggregate(self, round_idx):
        t = self.args.curr_train_iteration
        if "cfl" in self.args.concept_drift_algo_arg:
            if self.sc_state.cluster_cfl(t, round_idx + 1, self.bank, self.upload, self.upload_n):
                return self.get_global_model_params()  # skip: updates belong to an outdated set of models
        self._aggregate_models(np.any(self.sc_state.W[t] != 0, axis=1))
        if self.args.concept_drift_algo_arg == "hard-r":
            acc = self.evaluator.acc_matrix(list(range(self.bank.num_models)), t)
            self.sc_state.cluster(acc, t, round_idx + 1)
        return self.get_global_model_params()

    def extra_info(self, round_idx):
        return {"sc_weights": self.sc_state.get_weights()}

    def _route(self, c):
        t = self.args.curr_train_iteration
        m = self.sc_state.get_test_model_idx(t, c)
        return m, self.all_data[c][t], m, self.test_data_local_dicts[m].get(c)

    def _save_state(self):
        self.store.put("sc_state", self.sc_state)


class _ListEvaluator:
    """Evaluator over FedML list-of-batches data when no dense DriftData is attached."""

    def __init__(self, agg):
        self.agg = agg
        self.batch_size = agg.args.batch_size
        self.data = None

    def acc_matrix(self, model_ids, t):
        C = self.agg.args.client_num_in_total
        out = np.zeros((len(model_ids), C))
        for r, m in enumerate(model_ids):
            for c in range(C):
                k, n, _ = self.agg._infer(m, self.agg.all_data[c][t])
                out[r, c] = k / n if n else 0.0
        return out

    def pooled_acc(self, m, pairs, max_batches, rng):
        batches = [b for (c, t) in pairs for b in self.agg.all_data[c][t]]
        if not batches:
            return 0.0
        order = rng.permutation(len(batches))[: max_batches + 1]
        k, n, _ = self.agg._infer(m, [batches[i] for i in order])
        return k / n if n else 0.0


class FedAvgEnsAggregatorVanilla(_BaseAggregator):
    """Single-model FedAvg for ``exp``/``lin`` (parity: ``FedAvgEnsAggregatorVanilla.py``)."""

    def _route(self, c):
        return 0, self.train_data_local_dicts[0].get(c), 0, self.test_data_local_dicts[0].get(c)


class FedAvgEnsAggregatorAda(FedAvgEnsAggregatorVanilla):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.ada_state: AdaState = self.store.get("ada_state")
        mode = self.args.concept_drift_algo_arg.split("_")[1]
        if mode not in ("round", "iter"):
            raise NameError("ada config")
        self.update_each_round = mode == "round"

    def aggregate(self, round_idx):
        self._aggregate_models()
        a = self.args
        if self.update_each_round:
            self.ada_state.update(self.bank.theta[0], round_idx + a.curr_train_iteration * a.comm_round)
        elif round_idx == a.comm_round - 5:
            self.ada_state.update(self.bank.theta[0], a.curr_train_iteration)
        return self.get_global_model_params()

    def extra_info(self, round_idx):
        return {"lr": self.ada_state.current_lr()}

    def _save_state(self):
        self.store.put("ada_state", self.ada_state)


class FedAvgEnsAggregatorAue(_BaseAggregator):
    EPS = 1e-20
    per_client = False
    _report_test_loss = False

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        mser = (1 - 1.0 / self.class_num) ** 2
        w = np.full((self.args.client_num_in_total, self.bank.num_models), 1.0 / (mser + self.EPS))
        self.ens_weights = w / w.sum(1, keepdims=True)

    def update_ens_weights(self):
        mser, C, K = (1 - 1.0 / self.class_num) ** 2, self.args.client_num_in_total, self.bank.num_models
        sq, ns = np.zeros((K, C)), np.zeros(C)
        for k in range(1, K):
            for c in range(C):
                s, n = 0.0, 0
                for x, y in (self.train_data_local_dicts[0].get(c) or []):
                    with torch.no_grad():
                        s += float(ops.aue_sqerr(self.bank.forward(k, x.to(self.device)), y.to(self.device)))
                    n += y.shape[0]
                sq[k, c], ns[c] = s, n
        w = np.zeros((C, K))
        w[:, 0] = 1.0 / (mser + self.EPS)
        for k in range(1, K):
            if self.per_client:
                msei = np.where(ns > 0, sq[k] / np.maximum(ns, 1), 0.0)
            else:
                msei = np.full(C, sq[k].sum() / ns.sum() if ns.sum() > 0 else 0.0)
            w[:, k] = 1.0 / (mser + msei + self.EPS)
        self.ens_weights = w / w.sum(1, keepdims=True)

    def aggregate(self, round_idx):
        self._aggregate_models()
        if round_idx % 10 == 0 or round_idx > (self.args.comm_round - 10):
            self.update_ens_weights()
        return self.get_global_model_params()

    def _infer_ens(self, c, test_data):
        correct = total = 0.0
        w = torch.as_tensor(self.ens_weights[c], dtype=torch.float32, device=self.device)
        with torch.no_grad():
            for x, y in (test_data or []):
                x, y = x.to(self.device), y.to(self.device)
                preds = torch.stack([self.bank.forward(k, x).argmax(-1) for k in range(self.bank.num_models)])
                vote = ops.ensemble_vote(preds, w, self.class_num)
                correct += float((vote == y).sum())
                total += y.shape[0]
        return correct, total, 0.0

    def _test_client(self, c):
        tr = self._infer(0, self.train_data_local_dicts[0].get(c))
        return tr, self._infer_ens(c, self.test_data_local_dicts[0].get(c))


class FedAvgEnsAggregatorAuePc(FedAvgEnsAggregatorAue):
    per_client = True


class FedAvgEnsAggregatorKue(_BaseAggregator):
    _report_test_loss = False

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.kue_state: KueState = self.store.get("kue_state")
        if self.args.curr_train_iteration != 0:
            worst = self.kue_state.get_worst_idx()
            self.kue_state.initialize_mask(worst)
            self.bank.reinit(worst)
        self.ens_weights = np.ones(self.bank.num_models)

    def update_ens_weights(self):
        masks = self.kue_state.masks_tensor(self.device)
        for m in range(self.bank.num_models):
            A = torch.zeros(self.class_num, self.class_num, dtype=torch.float64)
            for c in range(self.args.client_num_in_total):
                for x, y in (self.train_data_local_dicts[m].get(c) or []):
                    x = x.to(self.device)
                    with torch.no_grad():
                        pred = self.bank.forward(m, x * masks[m].reshape((1,) + tuple(x.shape[1:]))).argmax(-1)
                    A += ops.confusion_matrix(pred, y.to(self.device), self.class_num).cpu()
            self.ens_weights[m] = ops.cohen_kappa(A)
        if self.args.curr_train_iteration != 0:
            self.kue_state.set_worst_idx(int(np.argmin(self.ens_weights)))

    def aggregate(self, round_idx):
        self._aggregate_models()
        if round_idx % 10 == 0 or round_idx > (self.args.comm_round - 10):
            self.update_ens_weights()
        return self.get_global_model_params()

    def extra_info(self, round_idx):
        return {"masks": self.kue_state.get_masks()}

    def _test_client(self, c):
        tr = self._infer(0, self.train_data_local_dicts[0].get(c))
        w = torch.as_tensor(self.ens_weights, dtype=torch.float32, device=self.device).clamp(min=0)
        w[self.kue_state.get_worst_idx()] = 0
        correct = total = 0.0
        with torch.no_grad():
            for x, y in (self.test_data_local_dicts[0].get(c) or []):
                x, y = x.to(self.device), y.to(self.device)
                probs = torch.stack([torch.softmax(self.bank.forward(m, x), 1) for m in range(self.bank.num_models)])
                correct += float((ops.soft_vote(probs, w) == y).sum())
                total += y.shape[0]
        return tr, (correct, total, 0.0)

    def _save_state(self):
        self.store.put("kue_state", self.kue_state)


class FedAvgEnsAggregatorDriftSurf(_BaseAggregator):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.ds_state: DriftSurfState = self.store.get("ds_state")
        a_ = self.args
        keys = list(self.ds_state.get_train_keys())
        if a_.curr_train_iteration != 0 and not a_.reset_models:
            for idx, key in enumerate(keys):
                snap = self.ds_state.snapshots.get(key)
                if snap is not None:
                    self.bank.theta[idx].copy_(snap.to(self.device))
        self.keys = keys
        self.test_model_idx = keys.index(self.ds_state.get_model_key()) if self.ds_state.get_model_key() in keys else 0

    def aggregate(self, round_idx):
        self._aggregate_models()
        if round_idx > (self.args.comm_round - 5):
            self._save_state()
        return self.get_global_model_params()

    def _route(self, c):
        m = self.test_model_idx
        return m, self.train_data_local_dicts[m].get(c), m, self.test_data_local_dicts[m].get(c)

    def _save_state(self):
        for idx, key in enumerate(self.keys):
            self.ds_state.set_snapshot(key, self.bank.theta[idx])
        self.store.put("ds_state", self.ds_state)


class FedAvgEnsAggregatorMultiModelAcc(_BaseAggregator):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.mm_state: MultiModelAccState = self.store.get("mm_state")

    def _route(self, c):
        mtr, mte = self.mm_state.get_train_model_idx(c), self.mm_state.get_test_model_idx(c)
        mtr, mte = min(mtr, self.bank.num_models - 1), min(mte, self.bank.num_models - 1)
        return mtr, self.train_data_local_dicts[mtr].get(c), mte, self.test_data_local_dicts[mte].get(c)

    def _after_client_eval(self, c, correct, n):
        if n:
            self.mm_state.set_acc(c, correct / n)

    def _save_state(self):
        self.store.put("mm_state", self.mm_state)


class FedAvgEnsAggregatorClusterFL(_BaseAggregator):
    """Legacy one-shot CFL (parity: ``FedAvgEnsAggregatorClusterFL.py:15-284``)."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.assign = [0] * self.args.client_num_in_total
        self.did_split = False

    def aggregate(self, round_idx):
        from .hclust import complete_linkage_bipartition
        if not self.did_split and round_idx == 100 and self.bank.num_models > 1:
            members = [c for c in range(self.worker_num) if self.assign[c] == 0 and float(self.upload_n[c, 0]) > 0]
            if len(members) >= 2:
                U = self.upload[members, 0, :] - self.bank.theta[0][None, :]
                S, norms = ops.gram_cosine(U)
                self.sink.log({"Max_Norm": float(norms.max()), "Mean_Norm": float(U.mean(0).norm()), "round": round_idx})
                _, g2 = complete_linkage_bipartition(S.cpu().numpy())
                for i in g2:
                    self.assign[members[i]] = 1
                self.bank.copy(1, 0)
                self.did_split = True
        self._aggregate_models()
        return self.get_global_model_params()

    def extra_info(self, round_idx):
        return list(self.assign)

    def _route(self, c):
        m = self.assign[c]
        return m, self.train_data_local_dicts[m].get(c), m, self.test_data_local_dicts[m].get(c)


# ====================================================================================== managers
class FedAvgEnsServerManager(ServerManager):
    """Round FSM (parity: ``FedAvgEnsServerManager.py:10-86``)."""

    def __init__(self, args, aggregator, comm=None, rank=0, size=0, backend="MPI"):
        super().__init__(args, comm, rank, size, backend)
        self.aggregator, self.round_num, self.round_idx = aggregator, args.comm_round, 0
        # logical workers may be PACKED onto fewer physical ranks (worker w lives on rank 1 + w % (size-1));
        # the reference needs one MPI rank per worker (FedAvgEnsAPI.py:86-92)
        self.worker_num = aggregator.worker_num
        # straggler tolerance (off unless args.round_timeout_s > 0): close a round with the uploads that arrived
        self.watchdog = RoundWatchdog(self, getattr(args, "round_timeout_s", 0.0), getattr(args, "min_workers_per_round", 1))
        self.dropped_uploads = 0

    def on_quiescent(self) -> bool:   # INPROC event loop: nothing more can arrive → treat as the round timeout
        return self.watchdog.fire_if_open()

    def _rank_of(self, worker: int) -> int:
        return 1 + worker % (self.size - 1)

    def send_init_msg(self):
        idx = self.aggregator.sample_round_clients(self.round_idx, self.args.client_num_in_total, self.args.client_num_per_round)
        params, extra = self.aggregator.get_global_model_params(), self.aggregator.extra_info(self.round_idx)
        for w in range(self.worker_num):
            self._send(MyMessage.MSG_TYPE_S2C_INIT_CONFIG, self._rank_of(w), params, idx[w], extra, w)
        self.watchdog.arm(self.round_idx)

    def register_message_receive_handlers(self):
        self.register_message_receive_handler(MyMessage.MSG_TYPE_C2S_SEND_MODEL_TO_SERVER,
                                              self.handle_message_receive_model_from_client)
        self.register_message_receive_handler(RoundWatchdog.MSG_TYPE_ROUND_TIMEOUT, self.handle_round_timeout)

    def handle_round_timeout(self, msg_params):
        """The watchdog fired: if round ``round_idx`` is still open and enough uploads arrived, close it without the
        stragglers (their weight is 0 in this round's aggregation)."""
        if int(msg_params.get("round_idx")) != self.round_idx or self.finished:
            return
        flags = self.aggregator.flag_client_model_uploaded_dict
        got = sum(1 for w in range(self.worker_num) if flags[w])
        if got < self.watchdog.min_workers:
            self.watchdog.arm(self.round_idx)      # keep waiting (threaded transports re-arm the timer)
            return
        missing = [w for w in range(self.worker_num) if not flags[w]]
        logging.warning("round %d: closing without workers %s (timeout)", self.round_idx, missing)
        self.watchdog.timeouts += 1
        self.args.watchdog_timeouts = getattr(self.args, "watchdog_timeouts", 0) + 1   # visible to the experiment driver
        for w in missing:
            self.aggregator.add_local_trained_result(w, {m: (None, 0) for m in range(self.aggregator.bank.num_models)})
        self.aggregator.check_whether_all_receive()
        self._complete_round()

    def handle_message_receive_model_from_client(self, msg_params):
        sender = msg_params.get(MyMessage.MSG_ARG_KEY_SENDER)
        worker = msg_params.get("worker_id")
        worker = sender - 1 if worker is None else int(worker)
        r = msg_params.get("round_idx")
        if r is not None and int(r) != self.round_idx:   # a straggler's upload for a round that was already closed
            self.dropped_uploads += 1
            return
        self.aggregator.add_local_trained_result(worker, msg_params.get(MyMessage.MSG_ARG_KEY_MODEL_AND_NUM_SAMPLES))
        if not self.aggregator.check_whether_all_receive():
            return
        self._complete_round()

    def _complete_round(self):
        self.watchdog.cancel()
        params = self.aggregator.aggregate(self.round_idx)
        self.aggregator.test_on_all_clients(self.round_idx)
        self.round_idx += 1
        if self.round_idx == self.round_num:
            self.save_model_params(params)
            self.finish()
            return
        idx = self.aggregator.sample_round_clients(self.round_idx, self.args.client_num_in_total, self.args.client_num_per_round)
        extra = self.aggregator.extra_info(self.round_idx)
        for w in range(self.worker_num):
            self._send(MyMessage.MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT, self._rank_of(w), params, idx[w], extra, w)
        self.watchdog.arm(self.round_idx)

    def _send(self, mtype, rid, params, client_index, extra, worker=None):
        msg = Message(mtype, self.get_sender_id(), rid)
        msg.add_params("worker_id", rid - 1 if worker is None else worker)
        msg.add_params(MyMessage.MSG_ARG_KEY_MODEL_PARAMS, params)
        msg.add_params(MyMessage.MSG_ARG_KEY_CLIENT_INDEX, str(client_index))
        msg.add_params(MyMessage.MSG_ARG_KEY_EXTRA_INFO, extra)
        self.send_message(msg)

    send_message_init_config = lambda self, rid, p, ci, ex: self._send(MyMessage.MSG_TYPE_S2C_INIT_CONFIG, rid, p, ci, ex)  # noqa: E731
    send_message_sync_model_to_client = lambda self, rid, p, ci, ex: self._send(MyMessage.MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT, rid, p, ci, ex)  # noqa: E731

    def save_model_params(self, params):
        store: StateStore = getattr(self.args, "state_store", None) or _default_store()
        bank = self.aggregator.bank
        store.put("model_params", {m: {k: v.detach().cpu().clone() for k, v in bank.state_dict(m).items()}
                                   for m in range(bank.num_models)})


class FedAvgEnsClientManager(ClientManager):
    """Client handlers (parity: ``FedAvgEnsClientManager.py:8-59``)."""

    def __init__(self, args, trainer, comm=None, rank=0, size=0, backend="MPI"):
        super().__init__(args, comm, rank, size, backend)
        # ``trainer`` may be a dict {worker_id: trainer} when several logical workers are packed on this rank
        self.trainers = trainer if isinstance(trainer, dict) else {rank - 1: trainer}
        self.trainer = next(iter(self.trainers.values()))
        self.num_rounds = args.comm_round
        self.rounds = {w: 0 for w in self.trainers}
        self.round_idx = 0

    def register_message_receive_handlers(self):
        self.register_message_receive_handler(MyMessage.MSG_TYPE_S2C_INIT_CONFIG, self.handle_message_init)
        self.register_message_receive_handler(MyMessage.MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT,
                                              self.handle_message_receive_model_from_server)

    def _update(self, msg_params) -> int:
        w = msg_params.get("worker_id")
        w = self.rank - 1 if w is None else int(w)
        tr = self.trainers[w]
        tr.update_model(msg_params.get(MyMessage.MSG_ARG_KEY_MODEL_PARAMS), msg_params.get(MyMessage.MSG_ARG_KEY_EXTRA_INFO))
        tr.update_dataset(int(msg_params.get(MyMessage.MSG_ARG_KEY_CLIENT_INDEX)))
        return w

    def handle_message_init(self, msg_params):
        w = self._update(msg_params)
        self.rounds[w] = self.round_idx = 0
        self._train(w)

    def handle_message_receive_model_from_server(self, msg_params):
        w = self._update(msg_params)
        self.rounds[w] += 1
        self.round_idx = self.rounds[w]
        self._train(w)
        if all(r == self.num_rounds - 1 for r in self.rounds.values()):
            self.finish()

    def send_model_to_server(self, receive_id, weights_and_num_samples, worker=None):
        msg = Message(MyMessage.MSG_TYPE_C2S_SEND_MODEL_TO_SERVER, self.get_sender_id(), receive_id)
        msg.add_params(MyMessage.MSG_ARG_KEY_MODEL_AND_NUM_SAMPLES, weights_and_num_samples)
        if worker is not None:
            msg.add_params("worker_id", worker)
            msg.add_params("round_idx", self.rounds.get(worker, self.round_idx))
        self.send_message(msg)

    def _train(self, w=None):
        w = next(iter(self.trainers)) if w is None else w
        # fault injection for tests / chaos runs: args.fault_drop = {round: [worker, ...]} — the worker trains but its
        # upload is lost (a crashed or partitioned client)
        drop = getattr(self.args, "fault_drop", None) or {}
        result = self.trainers[w].train()
        if w in drop.get(self.rounds.get(w, self.round_idx), ()):
            logging.warning("fault injection: dropping the upload of worker %d in round %d", w, self.rounds.get(w, 0))
            return
        self.send_model_to_server(0, result, w)


# ====================================================================================== API entry points
_AGGREGATORS = {
    "aue": FedAvgEnsAggregatorAue, "auepc": FedAvgEnsAggregatorAuePc, "driftsurf": FedAvgEnsAggregatorDriftSurf,
    "mmacc": FedAvgEnsAggregatorMultiModelAcc, "mmgeni": FedAvgEnsAggregatorMultiModelAcc,
    "mmgeniex": FedAvgEnsAggregatorMultiModelAcc, "clusterfl": FedAvgEnsAggregatorClusterFL,
    "softcluster": FedAvgEnsAggregatorSoftCluster, "softclusterwin-1": FedAvgEnsAggregatorSoftCluster,
    "softclusterreset": FedAvgEnsAggregatorSoftCluster, "ada": FedAvgEnsAggregatorAda,
    "exp": FedAvgEnsAggregatorVanilla, "lin": FedAvgEnsAggregatorVanilla, "kue": FedAvgEnsAggregatorKue,
}
_TRAINERS = {
    "clusterfl": FedAvgEnsTrainerClusterFL, "softcluster": FedAvgEnsTrainerSoftCluster,
    "softclusterwin-1": FedAvgEnsTrainerSoftCluster, "softclusterreset": FedAvgEnsTrainerSoftCluster,
    "ada": FedAvgEnsTrainerAda, "exp": FedAvgEnsTrainerExp, "lin": FedAvgEnsTrainerLin, "kue": FedAvgEnsTrainerKue,
}


def _unpack(datasets):
    cols = list(zip(*datasets))
    # (train_num, test_num, train_global, test_global, local_num_dict, train_local_dict, test_local_dict, class_num, feat)
    return dict(train_nums=list(cols[0]), test_nums=list(cols[1]), train_globals=list(cols[2]), test_globals=list(cols[3]),
                local_num=list(cols[4]), train_local=list(cols[5]), test_local=list(cols[6]))


def init_server(args, device, comm, rank, size, models, datasets, all_data, class_num, backend=None):
    d = _unpack(datasets)
    if args.concept_drift_algo not in _AGGREGATORS:
        raise NameError("concept_drift_algo")
    workers = int(getattr(args, "client_num_per_round", size - 1)) if getattr(args, "pack_workers", 0) else size - 1
    agg = _AGGREGATORS[args.concept_drift_algo](d["train_globals"], d["test_globals"], d["train_nums"], d["train_local"],
                                                d["test_local"], d["local_num"], all_data, workers, device, models,
                                                class_num, args)
    backend = backend or (comm.backend if hasattr(comm, "backend") else "MPI")
    mgr = FedAvgEnsServerManager(args, agg, comm.world if backend in ("INPROC", "STREAM") else comm, rank, size, backend)
    return mgr


def init_client(args, device, comm, process_id, size, models, datasets, all_local_data, backend=None):
    d = _unpack(datasets)
    cls = _TRAINERS.get(args.concept_drift_algo, FedAvgEnsTrainer)
    if getattr(args, "pack_workers", 0):  # all_local_data = all clients' data; host every worker w with 1 + w % (size-1) == rank
        trainer = {w: cls(w, d["train_local"], d["local_num"], d["train_nums"], all_local_data[w], device,
                          copy.deepcopy(models), args)
                   for w in range(int(args.client_num_per_round)) if 1 + w % (size - 1) == process_id}
    else:
        trainer = cls(process_id - 1, d["train_local"], d["local_num"], d["train_nums"], all_local_data, device, models, args)
    backend = backend or (comm.backend if hasattr(comm, "backend") else "MPI")
    return FedAvgEnsClientManager(args, trainer, comm.world if backend in ("INPROC", "STREAM") else comm, process_id, size, backend)


def FedML_FedAvgEns_distributed(process_id, worker_number, device, comm, models, datasets, all_data, class_num, args):
    """Rank 0 → server, rank k → client k-1 (parity: ``FedAvgEnsAPI.py:63-92``).  On the INPROC backend one call
    builds the server AND all clients (``models`` is then a factory or a list of per-rank model lists) and runs the
    deterministic event loop until the last round."""
    backend = comm.backend
    if backend in ("INPROC", "STREAM"):
        make = models if callable(models) else (lambda r: copy.deepcopy(models))
        server = init_server(args, device, comm, 0, worker_number, make(0), datasets, all_data, class_num, backend)
        clients = [init_client(args, device, comm, r, worker_number, make(r), datasets, all_data[r - 1], backend)
                   for r in range(1, worker_number)]
        mgrs = [server] + clients
        for m in mgrs:
            m.register_message_receive_handlers()
        server.send_init_msg()
        comm.world.run()
        return server
    if process_id == 0:
        server = init_server(args, device, comm, 0, worker_number, models, datasets, all_data, class_num, "DIST")
        server.send_init_msg()
        server.run()
        return server
    local = all_data if getattr(args, "pack_workers", 0) else all_data[process_id - 1]
    client = init_client(args, device, comm, process_id, worker_number, models, datasets, local, "DIST")
    client.run()
    return client
