"""Kernel-level timing of the persistent LSTM kernels (csrc/lstm_tc.cu): forward / BPTT time vs the number of concurrent
(pair, chunk) clusters, CUDA events, L2 flushed between timed launches, clocks recorded.  `--once N` runs ONE forward and ONE
backward launch with N clusters (for ncu)."""
import json
import sys

import torch

sys.path.insert(0, ".")
from bench import ClockSampler  # noqa: E402
from feddrift_b200.models.rnn import RNN_OriginalFedAvg  # noqa: E402
from feddrift_b200.models.utils import flat_spec, flatten_state_dict  # noqa: E402
from feddrift_b200.ops import lstm as L  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)
m = RNN_OriginalFedAvg()
spec = {k: off for k, _, _, off, _ in flat_spec(m)}
row = flatten_state_dict(m.state_dict()).to(dev)
keys = ["embeddings.weight", "lstm.weight_ih_l0", "lstm.weight_hh_l0", "lstm.bias_ih_l0", "lstm.bias_hh_l0", "lstm.weight_ih_l1",
        "lstm.weight_hh_l1", "lstm.bias_ih_l1", "lstm.bias_hh_l1"]
offs = [spec[k] for k in keys]
T = 80


def setup(n):
    arena = row.repeat(n)                                   # n independent parameter rows
    row_off = (torch.arange(n, device=dev) * row.numel()).long()
    tok = torch.randint(1, 90, (n, 16, T), device=dev, dtype=torch.int32)
    ws = L.Lstm2Workspace(n, T, dev, train=True)
    dh = torch.randn(n, 16, 256, device=dev) * 0.01
    return arena, row_off, tok, ws, dh


if len(sys.argv) > 2 and sys.argv[1] == "--once":
    n = int(sys.argv[2])
    arena, row_off, tok, ws, dh = setup(n)
    for _ in range(2):
        L.lstm2_pairs_forward(arena, row_off, offs, tok, 8, ws)
        L.lstm2_pairs_backward(arena, row_off, offs, tok, 8, ws, dh)
    torch.cuda.synchronize()
    sys.exit(0)

clk = ClockSampler(0)
clk.start()
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
res = []
for n in (1, 2, 16, 18, 32, 128):
    arena, row_off, tok, ws, dh = setup(n)
    for _ in range(3):
        L.lstm2_pairs_forward(arena, row_off, offs, tok, 8, ws)
        L.lstm2_pairs_backward(arena, row_off, offs, tok, 8, ws, dh)
    torch.cuda.synchronize()
    tf = tb = 0.0
    K = 5
    for i in range(K):
        flush.fill_(i)
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        L.lstm2_pairs_forward(arena, row_off, offs, tok, 8, ws)
        e1.record()
        L.lstm2_pairs_backward(arena, row_off, offs, tok, 8, ws, dh)
        e2.record()
        torch.cuda.synchronize()
        tf += e0.elapsed_time(e1)
        tb += e1.elapsed_time(e2)
    res.append({"clusters": n, "T": T, "fwd_ms": tf / K, "bwd_ms": tb / K, "fwd_us_per_timestep": tf / K / T * 1e3,
                "bwd_us_per_timestep": tb / K / T * 1e3})
    del arena, ws
    torch.cuda.empty_cache()
c = clk.stop()
for r in res:
    r["clocks"] = c
    print(json.dumps(r))
