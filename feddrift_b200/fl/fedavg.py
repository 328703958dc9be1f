"""Distributed single-model FedAvg and robust FedAvg (message-passing façade).

Parity: ``fedml_api/distributed/fedavg/*`` (FedAvgAPI, FedAVGAggregator, FedAVGTrainer, FedAvgServerManager,
FedAvgClientManager, utils, message_define — used by ``fedavg_cont_one`` for the ``win-k``/``all`` baselines and by
the mobile server) and ``fedml_api/distributed/fedavg_robust/*`` (norm-difference clipping + weak-DP noise).

Implementation: the multi-model ``fedavg_ens`` machinery with M = 1 — uploads land in a ``[workers, 1, P]`` arena,
aggregation is the K1 kernel; the robust variant clips every upload row around the global row with the fused
``ops.robust_clip_`` kernel (K10) and, for ``weak_dp``, adds Gaussian noise to the weight parameters before
averaging (the reference computes the noised tensor but sums the un-noised one —
``FedAvgRobustAggregator.py:96-105`` — that bug is not replicated).
"""
from __future__ import annotations

import copy
import logging
from typing import Dict, Optional

import numpy as np
import torch
from torch import nn

from .. import ops
from ..core.managers import ClientManager, RoundWatchdog, ServerManager
from ..core.message import Message
from ..core.robustness import RobustAggregator
from ..drift.fedavg_ens import _BaseAggregator
from ..models import utils as mutils


class MyMessage:
    MSG_TYPE_S2C_INIT_CONFIG = 1
    MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT = 2
    MSG_TYPE_C2S_SEND_MODEL_TO_SERVER = 3
    MSG_TYPE_C2S_SEND_STATS_TO_SERVER = 4
    MSG_ARG_KEY_TYPE = "msg_type"
    MSG_ARG_KEY_SENDER = "sender"
    MSG_ARG_KEY_RECEIVER = "receiver"
    MSG_ARG_KEY_NUM_SAMPLES = "num_samples"
    MSG_ARG_KEY_MODEL_PARAMS = "model_params"
    MSG_ARG_KEY_CLIENT_INDEX = "client_idx"


def transform_list_to_tensor(model_params_list: Dict) -> Dict:
    """JSON wire form → tensors (parity: ``fedavg/utils.py:5-8``)."""
    return {k: torch.from_numpy(np.asarray(v)).float() for k, v in model_params_list.items()}


def transform_tensor_to_list(model_params: Dict) -> Dict:
    return {k: v.detach().cpu().numpy().tolist() for k, v in model_params.items()}


class FedAVGTrainer:
    """Client trainer: the model stays on the device; ``epochs`` single-minibatch steps (list data) — parity
    ``FedAVGTrainer.py:10-80``.  ``full_epochs=True`` gives the robust variant's full passes
    (``FedAvgRobustTrainer.py:41-60``)."""

    def __init__(self, client_index, train_data_local_dict, train_data_local_num_dict, train_data_num, device, model, args,
                 full_epochs: bool = False):
        self.client_index = client_index
        self.train_data_local_dict, self.train_data_local_num_dict = train_data_local_dict, train_data_local_num_dict
        self.all_train_data_num = train_data_num
        self.device, self.args, self.model = device, args, model.to(device)
        self.full_epochs = full_epochs
        self.criterion = nn.CrossEntropyLoss().to(device)
        if args.client_optimizer == "sgd":
            self.optimizer = torch.optim.SGD(self.model.parameters(), lr=args.lr)
        else:
            self.optimizer = torch.optim.Adam(filter(lambda p: p.requires_grad, self.model.parameters()), lr=args.lr,
                                              weight_decay=args.wd, amsgrad=True)
        self.rng = np.random.RandomState(int(getattr(args, "dummy_arg", 0)) * 1000 + client_index + 1)
        self.update_dataset(client_index)

    def update_model(self, weights):
        if getattr(self.args, "is_mobile", 0) == 1:
            weights = transform_list_to_tensor(weights)
        self.model.load_state_dict(weights)

    def update_dataset(self, client_index):
        self.client_index = client_index
        self.train_local = self.train_data_local_dict.get(client_index)
        self.local_sample_number = self.train_data_local_num_dict.get(client_index, 0)

    def train(self):
        if self.local_sample_number == 0 or not self.train_local:
            return None, 0
        self.model.train()

        def step(x, labels):
            x, labels = x.to(self.device), labels.to(self.device)
            self.optimizer.zero_grad()
            self.criterion(self.model(x), labels).backward()
            self.optimizer.step()

        if self.full_epochs:
            for _ in range(self.args.epochs):
                for x, labels in self.train_local:
                    step(x, labels)
        elif isinstance(self.train_local, list):
            for _ in range(self.args.epochs):
                step(*self.train_local[self.rng.choice(len(self.train_local))])
        else:
            for _ in range(self.args.epochs):
                step(*next(iter(self.train_local)))
        weights = {k: v.detach().cpu() for k, v in self.model.state_dict().items()}
        if getattr(self.args, "is_mobile", 0) == 1:
            weights = transform_tensor_to_list(weights)
        return weights, self.local_sample_number


class FedAVGAggregator(_BaseAggregator):
    """Server side of single-model FedAvg (parity: ``FedAVGAggregator.py:13-178``)."""

    defend_uploads = False   # ``fedavg_robust`` applies its defense in ``_prepare_uploads``

    def __init__(self, train_global, test_global, all_train_data_num, train_data_local_dict, test_data_local_dict,
                 train_data_local_num_dict, worker_num, device, model, args):
        super().__init__([train_global], [test_global], [all_train_data_num], [train_data_local_dict], [test_data_local_dict],
                         [train_data_local_num_dict], None, worker_num, device, [model], None, args)
        self.model = self.models[0]
        self.train_data_local_dict, self.test_data_local_dict = train_data_local_dict, test_data_local_dict

    def get_global_model_params(self):
        sd = {k: v.detach().cpu().clone() for k, v in self.bank.state_dict(0).items()}
        return transform_tensor_to_list(sd) if getattr(self.args, "is_mobile", 0) == 1 else sd

    def add_local_trained_result(self, index, model_params, sample_num):  # noqa: D102 (FedAvg signature)
        super().add_local_trained_result(index, {0: (model_params, sample_num)})

    def _prepare_uploads(self) -> None:
        """Hook for defenses; operates on ``self.upload[:, 0, :]`` in place."""

    def aggregate(self, round_idx: Optional[int] = None):
        self._prepare_uploads()
        self._aggregate_models()
        return self.get_global_model_params()

    def _route(self, c):
        return 0, self.train_data_local_dict.get(c), 0, self.test_data_local_dict.get(c)


class FedAvgRobustAggregator(FedAVGAggregator):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.robust_aggregator = RobustAggregator(self.args)
        self.weight_mask = mutils.weight_param_mask(self.bank.spec).to(self.device)

    def _prepare_uploads(self) -> None:
        ra = self.robust_aggregator
        if ra.defense_type not in ("norm_diff_clipping", "weak_dp"):
            raise NotImplementedError("Non-supported Defense type ... ")
        rows = self.upload[:, 0, :]
        active = self.upload_n[:, 0] > 0
        if bool(active.any()):
            sel = rows[active]
            # clip + (weak_dp) Gaussian noise on the weight parameters in ONE fused pass (K10)
            self._noise_round = getattr(self, "_noise_round", 0) + 1
            std = float(ra.stddev) if ra.defense_type == "weak_dp" else 0.0
            ops.robust_clip_(sel, self.bank.theta[0], ra.norm_bound, self.weight_mask, std,
                             int(getattr(self.args, "dummy_arg", 0)) * 7919 + 77 + self._noise_round)
            rows[active] = sel


class FedAvgServerManager(ServerManager):
    """Round FSM (parity: ``FedAvgServerManager.py:21-77``); also the MQTT mobile server (``backend="MQTT"``)."""

    def __init__(self, args, aggregator, comm=None, rank=0, size=0, backend="MPI"):
        super().__init__(args, comm, rank, size, backend)
        self.aggregator, self.round_num, self.round_idx = aggregator, args.comm_round, 0
        # straggler tolerance (core.managers.RoundWatchdog; off unless args.round_timeout_s > 0) — mobile devices drop out
        self.watchdog = RoundWatchdog(self, getattr(args, "round_timeout_s", 0.0), getattr(args, "min_workers_per_round", 1))
        self.dropped_uploads = 0

    def on_quiescent(self) -> bool:
        return self.watchdog.fire_if_open()

    def send_init_msg(self):
        idx = self.aggregator.client_sampling(self.round_idx, self.args.client_num_in_total, self.args.client_num_per_round)
        params = self.aggregator.get_global_model_params()
        for pid in range(1, self.size):
            self.send_message_init_config(pid, params, idx[pid - 1])
        self.watchdog.arm(self.round_idx)

    def register_message_receive_handlers(self):
        self.register_message_receive_handler(MyMessage.MSG_TYPE_C2S_SEND_MODEL_TO_SERVER,
                                              self.handle_message_receive_model_from_client)
        self.register_message_receive_handler(RoundWatchdog.MSG_TYPE_ROUND_TIMEOUT, self.handle_round_timeout)

    def handle_round_timeout(self, msg_params):
        if int(msg_params.get("round_idx")) != self.round_idx or self.finished:
            return
        flags = self.aggregator.flag_client_model_uploaded_dict
        workers = range(self.size - 1)
        if sum(1 for w in workers if flags[w]) < self.watchdog.min_workers:
            self.watchdog.arm(self.round_idx)
            return
        missing = [w for w in workers if not flags[w]]
        logging.warning("round %d: closing without workers %s (timeout)", self.round_idx, missing)
        self.watchdog.timeouts += 1
        self.args.watchdog_timeouts = getattr(self.args, "watchdog_timeouts", 0) + 1
        for w in missing:
            self.aggregator.add_local_trained_result(w, None, 0)
        self.aggregator.check_whether_all_receive()
        self._complete_round()

    def handle_message_receive_model_from_client(self, msg_params):
        sender = int(msg_params.get(MyMessage.MSG_ARG_KEY_SENDER))
        r = msg_params.get("round_idx")
        if r is not None and int(r) != self.round_idx:   # upload of an already closed round
            self.dropped_uploads += 1
            return
        self.aggregator.add_local_trained_result(sender - 1, msg_params.get(MyMessage.MSG_ARG_KEY_MODEL_PARAMS),
                                                 msg_params.get(MyMessage.MSG_ARG_KEY_NUM_SAMPLES))
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
        idx = self.aggregator.client_sampling(self.round_idx, self.args.client_num_in_total, self.args.client_num_per_round)
        for rid in range(1, self.size):
            self.send_message_sync_model_to_client(rid, params, idx[rid - 1])
        self.watchdog.arm(self.round_idx)

    def _send(self, mtype, rid, params, client_index):
        msg = Message(mtype, self.get_sender_id(), rid)
        msg.add_params(MyMessage.MSG_ARG_KEY_MODEL_PARAMS, params)
        msg.add_params(MyMessage.MSG_ARG_KEY_CLIENT_INDEX, str(client_index))
        self.send_message(msg)

    def send_message_init_config(self, rid, params, client_index):
        self._send(MyMessage.MSG_TYPE_S2C_INIT_CONFIG, rid, params, client_index)

    def send_message_sync_model_to_client(self, rid, params, client_index):
        self._send(MyMessage.MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT, rid, params, client_index)

    def save_model_params(self, params):
        from ..drift.fedavg_ens import _default_store
        store = getattr(self.args, "state_store", None) or _default_store()
        store.put("model_params", {0: {k: torch.as_tensor(v) for k, v in params.items()}})


class FedAvgClientManager(ClientManager):
    def __init__(self, args, trainer, comm=None, rank=0, size=0, backend="MPI"):
        super().__init__(args, comm, rank, size, backend)
        self.trainer, self.num_rounds, self.round_idx = trainer, args.comm_round, 0

    def register_message_receive_handlers(self):
        self.register_message_receive_handler(MyMessage.MSG_TYPE_S2C_INIT_CONFIG, self.handle_message_init)
        self.register_message_receive_handler(MyMessage.MSG_TYPE_S2C_SYNC_MODEL_TO_CLIENT,
                                              self.handle_message_receive_model_from_server)

    def _update(self, msg_params):
        self.trainer.update_model(msg_params.get(MyMessage.MSG_ARG_KEY_MODEL_PARAMS))
        self.trainer.update_dataset(int(msg_params.get(MyMessage.MSG_ARG_KEY_CLIENT_INDEX)))

    def handle_message_init(self, msg_params):
        self._update(msg_params)
        self.round_idx = 0
        self._train()

    def handle_message_receive_model_from_server(self, msg_params):
        self._update(msg_params)
        self.round_idx += 1
        self._train()
        if self.round_idx == self.num_rounds - 1:
            self.finish()

    def send_model_to_server(self, receive_id, weights, local_sample_num):
        msg = Message(MyMessage.MSG_TYPE_C2S_SEND_MODEL_TO_SERVER, self.get_sender_id(), receive_id)
        msg.add_params(MyMessage.MSG_ARG_KEY_MODEL_PARAMS, weights)
        msg.add_params(MyMessage.MSG_ARG_KEY_NUM_SAMPLES, local_sample_num)
        msg.add_params("round_idx", self.round_idx)
        self.send_message(msg)

    def _train(self):
        w, n = self.trainer.train()
        drop = getattr(self.args, "fault_drop", None) or {}
        if (self.rank - 1) in drop.get(self.round_idx, ()):   # fault injection: this worker's upload is lost
            logging.warning("fault injection: dropping the upload of worker %d in round %d", self.rank - 1, self.round_idx)
            return
        self.send_model_to_server(0, w, n)


def FedML_FedAvg_distributed(process_id, worker_number, device, comm, model, train_data_num, train_data_global,
                             test_data_global, train_data_local_num_dict, train_data_local_dict, test_data_local_dict, args,
                             robust: bool = False):
    """Rank 0 → server, others → clients; INPROC comm builds everything in one process and runs the event loop
    (parity: ``FedAvgAPI.py`` / ``FedAvgRobustAPI.py``)."""
    backend = comm.backend
    agg_cls = FedAvgRobustAggregator if robust else FedAVGAggregator

    def server():
        agg = agg_cls(train_data_global, test_data_global, train_data_num, train_data_local_dict, test_data_local_dict,
                      train_data_local_num_dict, worker_number - 1, device, copy.deepcopy(model), args)
        return FedAvgServerManager(args, agg, comm.world if backend in ("INPROC", "STREAM") else comm, 0, worker_number,
                                   backend if backend in ("INPROC", "STREAM", "MQTT") else "DIST")

    def client(rank):
        tr = FedAVGTrainer(rank - 1, train_data_local_dict, train_data_local_num_dict, train_data_num, device,
                           copy.deepcopy(model), args, full_epochs=robust)
        return FedAvgClientManager(args, tr, comm.world if backend in ("INPROC", "STREAM") else comm, rank, worker_number,
                                   backend if backend in ("INPROC", "STREAM", "MQTT") else "DIST")

    if backend in ("INPROC", "STREAM"):
        srv = server()
        mgrs = [srv] + [client(r) for r in range(1, worker_number)]
        for m in mgrs:
            m.register_message_receive_handlers()
        srv.send_init_msg()
        comm.world.run()
        return srv
    if process_id == 0:
        srv = server()
        srv.send_init_msg()
        srv.run()
        return srv
    c = client(process_id)
    c.run()
    return c


def FedML_FedAvgRobust_distributed(*a, **k):
    return FedML_FedAvg_distributed(*a, robust=True, **k)
