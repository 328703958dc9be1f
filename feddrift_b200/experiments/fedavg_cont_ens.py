"""``main_fedavg.py`` of ``fedml_experiments/distributed/fedavg_cont_ens`` re-imagined: ONE process (or one torchrun
job) runs the whole continual experiment — data preparation, every time step, checkpointing — instead of a bash
loop that relaunches ``mpirun`` per time step (``run_fedavg_distributed_pytorch.sh:49-84``).

  # device engine (default; fused sm_90a round kernel when the model is a small MLP)
  python -m feddrift_b200.experiments.fedavg_cont_ens --dataset sea --model fnn --concept_drift_algo softcluster \\
      --concept_drift_algo_arg H_A_C_1_10_0 --change_points A --comm_round 200 --total_train_iteration 10

  # FedML message-passing façade (reference-compatible managers/aggregators/trainers), in-process or gloo
  python -m feddrift_b200.experiments.fedavg_cont_ens --engine facade --backend INPROC ...
  torchrun --nproc-per-node 11 --master-addr 127.0.0.1 -m feddrift_b200.experiments.fedavg_cont_ens --engine facade --backend GLOO ...

Positional-argument compatibility with the reference's run script is provided by ``run_fedavg_distributed.sh``.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
import random

import numpy as np
import torch


def add_args(parser: argparse.ArgumentParser) -> argparse.ArgumentParser:
    """Same flags/defaults as the reference ``main_fedavg.py:42-139`` + ``prepare_data.py`` + engine selection."""
    a = parser.add_argument
    a("--model", type=str, default="fnn"); a("--dataset", type=str, default="sea")
    a("--data_dir", type=str, default=None)
    a("--client_num_in_total", type=int, default=10); a("--client_num_per_round", type=int, default=10)
    a("--batch_size", type=int, default=500); a("--client_optimizer", type=str, default="adam")
    a("--lr", type=float, default=0.01); a("--wd", type=float, default=0.001)
    a("--epochs", type=int, default=5); a("--comm_round", type=int, default=200)
    a("--is_mobile", type=int, default=0); a("--frequency_of_the_test", type=int, default=1)
    a("--gpu_server_num", type=int, default=1); a("--gpu_num_per_server", type=int, default=1)
    a("--ci", type=int, default=0)
    a("--total_train_iteration", type=int, default=10); a("--curr_train_iteration", type=int, default=0)
    a("--drift_together", type=int, default=0); a("--report_client", type=int, default=1)
    a("--retrain_data", type=str, default="win-1")
    a("--concept_drift_algo", type=str, default="softcluster"); a("--concept_drift_algo_arg", type=str, default="H_A_C_1_10_0")
    a("--ensemble_window", type=int, default=4); a("--concept_num", type=int, default=4)
    a("--change_points", type=str, default="A"); a("--time_stretch", type=int, default=1)
    a("--reset_models", type=int, default=0); a("--noise_prob", type=float, default=0.0)
    a("--dummy_arg", type=int, default=0); a("--sample_num", type=int, default=100)
    a("--engine", type=str, default="device", choices=["device", "facade"])
    a("--backend", type=str, default="INPROC", choices=["INPROC", "GLOO", "NCCL"])
    a("--device", type=str, default=None); a("--checkpoint_dir", type=str, default=None)
    a("--resume", type=int, default=0); a("--metrics_file", type=str, default=None)
    a("--use_wandb", type=int, default=0); a("--strict_ref", type=int, default=0)
    a("--rounds_per_launch", type=int, default=0)
    # server optimizer on every cluster model (FedOpt per slot; flag names as in `main.py fedopt`), single-GPU
    a("--server_optimizer", type=str, default="none", choices=["none", "sgd", "adam", "adagrad", "yogi"])
    a("--server_lr", type=float, default=1.0); a("--server_momentum", type=float, default=0.0)
    a("--server_eps", type=float, default=1e-8, help="τ of adam / adagrad / yogi")
    # robust aggregation of every upload before its cluster average (flag names as in `main.py fedavg_robust`); weak_dp is
    # the reference's backdoor defense (clipping + Gaussian noise) and carries no (ε, δ) privacy guarantee
    a("--defense_type", type=str, default="none", choices=["none", "norm_diff_clipping", "weak_dp"])
    a("--norm_bound", type=float, default=5.0); a("--stddev", type=float, default=0.025, help="weak_dp noise stddev")
    # compression of every upload against its round-start cluster model, before the raw-update hooks, the defense and the
    # average: unbiased stochastic quantization (qsgd; s levels per sign, one max-norm scale per bucket of b entries) or
    # top-k sparsification with error feedback (eftopk; the ρ·n largest entries of update + residual are sent, the rest is
    # carried to the client's next upload)
    a("--compression", type=str, default="none", choices=["none", "qsgd", "eftopk"])
    a("--quantize_level", type=int, default=16, help="QSGD levels s, 1..65535 (s = 1: ternary)")
    a("--quantize_bucket", type=int, default=512, help="QSGD bucket size b (entries per scale), >= 1")
    a("--topk_ratio", type=float, default=0.01, help="eftopk: fraction ρ of the trainable entries kept, 0 < ρ <= 1")
    # Byzantine-robust cluster aggregation (Yin et al., 2018): the coordinate-wise median or β-trimmed mean of the slot's
    # uploads (after compression and the defense), each participant counted once, instead of the weighted average
    a("--aggregation_rule", type=str, default="mean",
      choices=["mean", "median", "trimmed_mean", "geometric_median", "multi_krum", "centered_clip"])
    a("--trim_ratio", type=float, default=0.1, help="trimmed_mean: fraction β dropped at each end, 0 <= β < 0.5")
    # geometric median (RFA, Pillutla et al.): smoothed Weiszfeld steps from the coordinate-wise median
    a("--geomed_iters", type=int, default=4, help="geometric_median: Weiszfeld iterations R, 1..100")
    a("--geomed_nu", type=float, default=1e-6, help="geometric_median: smoothing ν > 0 (weights 1 / max(ν, distance))")
    # Multi-Krum (Blanchard et al., 2017): the average of the m uploads closest to their n − f − 2 nearest neighbours; one
    # rule with one name, --krum_m 1 is plain Krum
    a("--krum_f", type=int, default=1, help="multi_krum: Byzantine uploads f assumed per slot, 0..65535")
    a("--krum_m", type=int, default=1, help="multi_krum: uploads m averaged, 1..65535 (1: Krum)")
    # centered clipping (Karimireddy, He & Jaggi, 2021): every update is clipped to radius τ around the slot's previous
    # aggregate and the clipped updates are averaged, L times; the center is reset at every time step
    a("--cclip_tau", type=float, default=1.0, help="centered_clip: clipping radius τ > 0")
    a("--cclip_iters", type=int, default=1, help="centered_clip: clipping iterations L, 1..100")
    # simulated Byzantine clients: a fixed set of --attack_clients clients poisons its uploads after compression (sign_flip:
    # the reversed update, gaussian: noise around the model, alie: "A Little Is Enough", ipm: inner-product manipulation)
    a("--attack_type", type=str, default="none", choices=["none", "sign_flip", "gaussian", "alie", "ipm"])
    a("--attack_clients", type=int, default=0, help="attack: number a of Byzantine clients, 0..client_num_in_total")
    a("--attack_scale", type=float, default=1.0, help="attack: strength s > 0 (sign_flip / gaussian scale, ALIE z, IPM ε)")
    # FedProx local training: every client step minimises CE + mu/2‖w − w_m‖², w_m the cluster model it received (0 = off)
    a("--fedprox_mu", type=float, default=0.0)
    # façade extras: worker packing, zero-copy device payloads, straggler tolerance (core.managers.RoundWatchdog)
    a("--pack_workers", type=int, default=0); a("--zero_copy", type=int, default=0)
    a("--round_timeout_s", type=float, default=0.0, help="> 0: close a round without workers whose upload did not arrive in time")
    a("--min_workers_per_round", type=int, default=1)
    return parser


def seed_everything(seed: int) -> None:
    from ..models import utils as mutils
    np.random.seed(seed); torch.manual_seed(seed); random.seed(seed)
    mutils.torch_seed = seed


def run_device(args, sink):
    from ..sim import DriftSim
    from ..sim import checkpoint as ckpt
    sim = DriftSim(args, device=args.device, sink=sink)
    start = 0
    if args.resume and args.checkpoint_dir and ckpt.latest(args.checkpoint_dir):
        start = ckpt.resume(sim, ckpt.latest(args.checkpoint_dir))
    out = sim.run(start_iteration=start)
    ckpt.export_model_params(sim, os.path.join(args.checkpoint_dir or ".", "model_params.pt")) if args.checkpoint_dir else None
    return out


def run_facade(args, sink):
    """Time-step loop over the FedML-compatible message-passing stack."""
    from ..data.drift import generate_drift_data, load_all_data, load_partition_data
    from ..drift.fedavg_ens import (FedML_FedAvgEns_data_loader, FedML_FedAvgEns_distributed, FedML_init, StateStore)
    from ..models.utils import create_model
    size = args.client_num_per_round + 1
    comm, process_id, worker_number = FedML_init(args.backend, size)
    data = generate_drift_data(args.dataset, args.total_train_iteration, args.client_num_in_total, args.sample_num,
                               args.noise_prob, args.time_stretch, args.change_points, bool(args.drift_together), seed=0,
                               data_dir=args.data_dir)
    args.state_store = StateStore(args.checkpoint_dir)
    args.drift_data = data
    device = torch.device(args.device or "cpu")
    history = []
    for t in range(args.total_train_iteration):
        args.curr_train_iteration = t
        seed_everything(args.dummy_arg)

        def loader(a):
            tup = load_partition_data(data, a.batch_size, a.curr_train_iteration, a.retrain_data)
            return list(tup[1:]) + [data.feature_num]
        bank = ev = None
        if t > 0 and args.concept_drift_algo in ("mmacc", "driftsurf"):
            # these algorithms score last step's models on the new data BEFORE choosing training sets
            from ..drift.evaluator import Evaluator
            from ..parallel.arena import ModelBank
            prev_params = args.state_store.get("model_params") or {}
            bank = ModelBank(create_model(args.model, data.class_num, data.feature_num), len(prev_params) + 1, device)
            for m, p in prev_params.items():
                bank.load_state_dict(m, p)
            ev = Evaluator(bank, data.to(device), args.batch_size)
        datasets = FedML_FedAvgEns_data_loader(args, loader, device, comm, process_id, bank=bank, evaluator=ev)
        all_data = load_all_data(data, args.batch_size, t)
        class_num, feat = datasets[0][-2], datasets[0][-1]
        models = [create_model(args.model, class_num, feat) for _ in datasets]
        prev = args.state_store.get("model_params") if (t > 0 and not args.reset_models) else None
        if prev is not None:
            if args.concept_drift_algo in ("aue", "auepc"):
                for m in range(1, len(models)):
                    models[m].load_state_dict(prev[m - 1])
            elif args.concept_drift_algo != "driftsurf":
                for m, p in prev.items():
                    if m < len(models):
                        models[m].load_state_dict(p)
        server = FedML_FedAvgEns_distributed(process_id, worker_number, device, comm, models, datasets, all_data,
                                             class_num, args)
        if process_id == 0:
            history.append({"iteration": t, "train_acc": sink.last("Train/Acc"), "test_acc": sink.last("Test/Acc")})
    if args.backend in ("GLOO", "NCCL"):
        from ..drift.fedavg_ens import FedML_finalize
        FedML_finalize()
    return {"history": history, "summary": dict(sink.run.summary)}


def main(argv=None):
    args = add_args(argparse.ArgumentParser()).parse_args(argv)
    logging.basicConfig(level=logging.WARNING)
    from ..utils.metrics import MetricsSink, set_sink
    sink = set_sink(MetricsSink(args.metrics_file, use_wandb=bool(args.use_wandb)))
    sink.init(project="fedml", name=f"FedAvgCont(d)-{args.dataset}-r{args.comm_round}-e{args.epochs}-lr{args.lr}"
                                      f"-{args.concept_drift_algo}", config=args)
    seed_everything(args.dummy_arg)
    out = run_device(args, sink) if args.engine == "device" else run_facade(args, sink)
    sink.finish()
    last = out["history"][-1] if out["history"] else {}
    print(json.dumps({"final": last, "summary": out["summary"]}, default=str))
    return out


if __name__ == "__main__":
    main()
