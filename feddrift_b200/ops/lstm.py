"""Fused 2-layer LSTM(256) — Python side of ``csrc/lstm_tc.cu`` (persistent 8-CTA cluster kernel, mma.sync).

Reference semantics: ``nn.Embedding(V, E) → nn.LSTM(E, 256, num_layers=2, batch_first=True)`` as used by
``RNN_OriginalFedAvg`` (``fedml_api/model/nlp/rnn.py:18-33``); the reference runs it through cuDNN's per-timestep kernels.

* ``lstm2_embed_forward(tokens, emb, lstm_params, need_all)`` is an autograd function: ONE kernel launch runs the whole
  sequence (all T steps, both layers) for every 16-row batch chunk, ONE launch runs BPTT, and the weight gradients are
  five GEMMs over the saved bf16 histories (``dW = dGᵀ·H`` on the MN-major wgmma GEMM).
* ``Lstm2Workspace`` / ``lstm2_pairs_forward`` / ``lstm2_pairs_backward`` expose the many-pairs-per-launch form used by the
  batched federated executor: every (client, model) pair is one thread-block cluster reading its weights straight from its
  ``ClientArena`` row (no parameter copies).

Compute: bf16 operands, fp32 accumulation / cell state / gates.  CPU tensors and unsupported shapes fall back to the
plain PyTorch modules (which are also the numerics oracle of ``tests/test_gpu_lstm.py``).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _ext

H = 256
NB = 16
CALLS = {"fwd": 0, "bwd": 0}   # tests assert the native path is live

PARAM_ORDER = ("emb", "w_ih1", "w_hh1", "b_ih1", "b_hh1", "w_ih2", "w_hh2", "b_ih2", "b_hh2")


def eligible(tokens: torch.Tensor, emb: torch.Tensor, lstm: torch.nn.LSTM) -> bool:
    import os
    if os.environ.get("FDB_NO_FUSED_LSTM") == "1":   # numerics oracle / A-B switch: plain nn.LSTM (cuDNN)
        return False
    return bool(tokens.is_cuda and emb.is_cuda and lstm.hidden_size == H and lstm.num_layers == 2 and lstm.batch_first
                and not lstm.bidirectional and lstm.bias and lstm.proj_size == 0 and emb.shape[1] <= 16 and tokens.dim() == 2
                and float(getattr(lstm, "dropout", 0.0)) == 0.0 and _ext.available() and hasattr(_ext.load(), "lstm2_forward"))


def _flat_params(tensors: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, List[int]]:
    """(flat fp32 arena, element offsets).  When every tensor is a contiguous view of ONE storage (bank-bound modules:
    parameters are views of a ``ClientArena`` / graph row) the storage itself is the arena — no copy."""
    t0 = tensors[0]
    st = t0.untyped_storage()
    same = all(t.is_contiguous() and t.dtype == torch.float32 and t.untyped_storage().data_ptr() == st.data_ptr() for t in tensors)
    if same:
        flat = torch.empty(0, dtype=torch.float32, device=t0.device).set_(st)
        return flat, [int(t.storage_offset()) for t in tensors]
    offs, chunks, o = [], [], 0
    for t in tensors:
        offs.append(o)
        n = t.numel()
        pad = (-n) % 4          # keep every tensor 16-byte aligned (vectorised weight loads)
        chunks.append(t.detach().reshape(-1).float())
        if pad:
            chunks.append(torch.zeros(pad, dtype=torch.float32, device=t.device))
        o += n + pad
    return torch.cat(chunks), offs


class Lstm2Workspace:
    """History buffers of ``npairs`` concurrent sequences (16 rows each) of length T.  Layout is LAYER-outermost
    (``[2, npairs, T, 16, …]``) so that one layer's rows of all pairs form one ``[npairs·T·16, 1024]`` matrix for the
    (batched) weight-gradient GEMMs.  ``train=False`` keeps no history (inference: only ``hlast``)."""

    def __init__(self, npairs: int, T: int, device, train: bool = True, keep_h: Optional[bool] = None):
        self.npairs, self.T = int(npairs), int(T)
        keep_h = train if keep_h is None else keep_h
        self.gates = torch.empty(2, npairs, T, NB, 4 * H, dtype=torch.float32, device=device) if train else None
        self.cst = torch.empty(2, npairs, T, NB, H, dtype=torch.float32, device=device) if train else None
        self.hhist = torch.zeros(2, npairs, T + 1, NB, H, dtype=torch.bfloat16, device=device) if keep_h else None  # [:, :, 0] = h_{-1} = 0
        self.hlast = torch.empty(npairs, NB, H, dtype=torch.float32, device=device)
        self.dgates = torch.empty(2, npairs, T, NB, 4 * H, dtype=torch.bfloat16, device=device) if train else None


def lstm2_pairs_forward(arena: torch.Tensor, row_off: torch.Tensor, offs: Sequence[int], tokens: torch.Tensor, E: int,
                        ws: Lstm2Workspace) -> None:
    """tokens: int32 ``[npairs, 16, T]``; row_off: int64 ``[npairs]`` element offsets of the pairs' parameter rows in ``arena``."""
    CALLS["fwd"] += 1
    _ext.load(required=True).lstm2_forward(arena, row_off, [int(o) for o in offs], tokens, ws.gates, ws.cst, ws.hhist, ws.hlast, int(E))


def lstm2_pairs_backward(arena: torch.Tensor, row_off: torch.Tensor, offs: Sequence[int], tokens: torch.Tensor, E: int,
                         ws: Lstm2Workspace, dh2_last: Optional[torch.Tensor], dh2_all: Optional[torch.Tensor] = None) -> None:
    CALLS["bwd"] += 1
    _ext.load(required=True).lstm2_backward(arena, row_off, [int(o) for o in offs], tokens, ws.gates, ws.cst, ws.hhist, ws.hlast, int(E),
                                            dh2_last, dh2_all, ws.dgates)


def lstm2_weight_grads(ws: Lstm2Workspace, tokens: torch.Tensor, emb: torch.Tensor, w_ih1: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Parameter gradients when ALL chunks of the workspace share one parameter set (the autograd-module path)."""
    ext = _ext.load(required=True)
    T, n = ws.T, ws.npairs
    dG1 = ws.dgates[0].reshape(n * T * NB, 4 * H)                # contiguous views
    dG2 = ws.dgates[1].reshape(n * T * NB, 4 * H)
    H1prev = ws.hhist[0, :, :T].reshape(n * T * NB, H)
    H1cur = ws.hhist[0, :, 1:].reshape(n * T * NB, H)
    H2prev = ws.hhist[1, :, :T].reshape(n * T * NB, H)
    g: Dict[str, torch.Tensor] = {}
    # dW[1024, 256] = dGᵀ · H: both operands are consumed MN-major ([reduction, rows] row-major) — no transposes
    g["w_hh1"] = ext.gemm_bias_act(dG1, H1prev.contiguous(), True, True, None, False, True)
    g["w_ih2"] = ext.gemm_bias_act(dG2, H1cur.contiguous(), True, True, None, False, True)
    g["w_hh2"] = ext.gemm_bias_act(dG2, H2prev.contiguous(), True, True, None, False, True)
    dG1f, dG2f = dG1.float(), dG2.float()
    g["b_ih1"] = g["b_hh1"] = dG1f.sum(0)
    g["b_ih2"] = g["b_hh2"] = dG2f.sum(0)
    tok = tokens.long().permute(0, 2, 1).reshape(-1)            # [n, T, 16] order of the history rows
    X = emb.detach()[tok].to(torch.bfloat16).float()            # the kernel fed bf16 embeddings to the tensor core
    g["w_ih1"] = dG1f.t() @ X                                    # [1024, E]
    dX = dG1f @ w_ih1.detach().to(torch.bfloat16).float()        # [n·T·16, E]
    ge = torch.zeros_like(emb, dtype=torch.float32)
    ge.index_add_(0, tok, dX)
    g["emb"] = ge
    return g


def lstm2_weight_grads_per_chunk(ws: Lstm2Workspace) -> Dict[str, torch.Tensor]:
    """Per-chunk recurrent weight gradients ``[nchunks, 1024, 256]`` in ONE batched wgmma GEMM launch per matrix (every
    chunk is a batch entry with its own reduction rows); falls back to a loop when ``T·16`` is not a multiple of 64."""
    ext = _ext.load(required=True)
    T, n = ws.T, ws.npairs
    K = T * NB
    dG1 = ws.dgates[0].reshape(n * K, 4 * H)
    dG2 = ws.dgates[1].reshape(n * K, 4 * H)
    hh1 = ws.hhist[0].reshape(n * (T + 1) * NB, H)
    hh2 = ws.hhist[1].reshape(n * (T + 1) * NB, H)
    hs = (T + 1) * NB
    if K % 64 == 0:
        return {"w_hh1": ext.gemm_batched_mn(dG1, hh1, K, n, 0, K, 0, hs),
                "w_ih2": ext.gemm_batched_mn(dG2, hh1, K, n, 0, K, NB, hs),
                "w_hh2": ext.gemm_batched_mn(dG2, hh2, K, n, 0, K, 0, hs)}
    out = {k: [] for k in ("w_hh1", "w_ih2", "w_hh2")}
    for i in range(n):
        a1, a2 = dG1[i * K:(i + 1) * K], dG2[i * K:(i + 1) * K]
        out["w_hh1"].append(ext.gemm_bias_act(a1, hh1[i * hs:i * hs + K], True, True, None, False, True))
        out["w_ih2"].append(ext.gemm_bias_act(a2, hh1[i * hs + NB:i * hs + NB + K], True, True, None, False, True))
        out["w_hh2"].append(ext.gemm_bias_act(a2, hh2[i * hs:i * hs + K], True, True, None, False, True))
    return {k: torch.stack(v) for k, v in out.items()}


def lstm_head(arena: torch.Tensor, row_off: torch.Tensor, off_fcw: int, off_fcb: int, hlast: torch.Tensor, labels: torch.Tensor,
              scale: torch.Tensor, V: int):
    """fc + softmax-CE + every head gradient for all chunks in one launch → (dh [n,16,256], dW [n,V,256], db [n,V], loss [n])."""
    n = row_off.numel()
    dev = hlast.device
    dh = torch.empty(n, NB, H, dtype=torch.float32, device=dev)
    dW = torch.empty(n, V, H, dtype=torch.float32, device=dev)
    db = torch.empty(n, V, dtype=torch.float32, device=dev)
    loss = torch.empty(n, dtype=torch.float32, device=dev)
    _ext.load(required=True).lstm_head(arena, row_off, int(off_fcw), int(off_fcb), hlast, labels, scale, dh, dW, db, loss, int(V))
    return dh, dW, db, loss


class _Lstm2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tokens, need_all, padding_idx, emb, w_ih1, w_hh1, b_ih1, b_hh1, w_ih2, w_hh2, b_ih2, b_hh2):
        B, T = tokens.shape
        E = emb.shape[1]
        dev = tokens.device
        tensors = (emb, w_ih1, w_hh1, b_ih1, b_hh1, w_ih2, w_hh2, b_ih2, b_hh2)
        arena, offs = _flat_params([t.detach() for t in tensors])
        n = (B + NB - 1) // NB
        tok = torch.zeros(n * NB, T, dtype=torch.int32, device=dev)
        tok[:B] = tokens.to(torch.int32)
        tok = tok.reshape(n, NB, T)
        row_off = torch.zeros(n, dtype=torch.int64, device=dev)
        train = any(ctx.needs_input_grad[3:])   # (grad mode is always off inside Function.forward)
        ws = Lstm2Workspace(n, T, dev, train=train, keep_h=train or bool(need_all))
        lstm2_pairs_forward(arena, row_off, offs, tok, E, ws)
        ctx.ws, ctx.tok, ctx.offs, ctx.arena, ctx.row_off = ws, tok, offs, arena, row_off
        ctx.B, ctx.T, ctx.E, ctx.need_all, ctx.padding_idx = B, T, E, bool(need_all), padding_idx
        ctx.save_for_backward(emb, w_ih1)
        if need_all:   # [B, T, 256] (bf16-rounded hidden states, exactly what the next timestep consumed)
            return ws.hhist[1, :, 1:].permute(0, 2, 1, 3).reshape(n * NB, T, H)[:B].float()
        return ws.hlast.reshape(n * NB, H)[:B].clone()

    @staticmethod
    def backward(ctx, gout):
        emb, w_ih1 = ctx.saved_tensors
        ws, B, T, n = ctx.ws, ctx.B, ctx.T, ctx.ws.npairs
        dev = gout.device
        if ctx.need_all:
            d = torch.zeros(n * NB, T, H, dtype=torch.float32, device=dev)
            d[:B] = gout.float()
            dh_all = d.reshape(n, NB, T, H).permute(0, 2, 1, 3).contiguous()    # [n, T, 16, 256]
            lstm2_pairs_backward(ctx.arena, ctx.row_off, ctx.offs, ctx.tok, ctx.E, ws, None, dh_all)
        else:
            d = torch.zeros(n * NB, H, dtype=torch.float32, device=dev)
            d[:B] = gout.float()
            lstm2_pairs_backward(ctx.arena, ctx.row_off, ctx.offs, ctx.tok, ctx.E, ws, d.reshape(n, NB, H), None)
        g = lstm2_weight_grads(ws, ctx.tok, emb, w_ih1)
        if ctx.padding_idx is not None:
            g["emb"][ctx.padding_idx] = 0
        ctx.ws = None
        return (None, None, None, g["emb"], g["w_ih1"], g["w_hh1"], g["b_ih1"], g["b_hh1"], g["w_ih2"], g["w_hh2"], g["b_ih2"], g["b_hh2"])


def lstm2_embed_forward(tokens: torch.Tensor, embedding: torch.nn.Embedding, lstm: torch.nn.LSTM, need_all: bool = False) -> torch.Tensor:
    """``lstm(embedding(tokens))``: the last hidden state ``[B, 256]`` (or all ``[B, T, 256]`` with ``need_all``) through the
    fused kernel.  Caller checks :func:`eligible`."""
    return _Lstm2Fn.apply(tokens, need_all, embedding.padding_idx, embedding.weight, lstm.weight_ih_l0, lstm.weight_hh_l0,
                          lstm.bias_ih_l0, lstm.bias_hh_l0, lstm.weight_ih_l1, lstm.weight_hh_l1, lstm.bias_ih_l1, lstm.bias_hh_l1)
