"""Robust aggregation defenses (norm-difference clipping, weak DP noise).

Parity: ``fedml_core/robustness/robust_aggregation.py:4-55``.  On CUDA the flat
variants (`clip_flat`) run the fused ``ops.robust_clip_`` kernel over arena
rows (norm + clip (+ Philox noise) in one pass, K10 in SURVEY §2.9); the
state_dict API below is the drop-in compatible surface.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch


def is_weight_param(k: str) -> bool:
    return "running_mean" not in k and "running_var" not in k and "num_batches_tracked" not in k


def vectorize_weight(state_dict: Dict[str, torch.Tensor]) -> torch.Tensor:
    return torch.cat([v.reshape(-1).float() for k, v in state_dict.items() if is_weight_param(k)])


def load_model_weight_diff(local_state_dict, weight_diff: torch.Tensor, global_state_dict):
    """w_global + clipped(w_local - w_global) on weight params; BN statistics pass through."""
    sd = local_state_dict.state_dict() if hasattr(local_state_dict, "state_dict") and not isinstance(
        local_state_dict, dict) else local_state_dict
    out, off = {}, 0
    for k, v in sd.items():
        if is_weight_param(k):
            n = v.numel()
            out[k] = weight_diff[off:off + n].view(v.size()).to(v.dtype) + global_state_dict[k]
            off += n
        else:
            out[k] = v
    return out


class RobustAggregator:
    def __init__(self, args):
        self.defense_type = getattr(args, "defense_type", "norm_diff_clipping")
        self.norm_bound = float(getattr(args, "norm_bound", 5.0))
        self.stddev = float(getattr(args, "stddev", 0.025))

    def norm_diff_clipping(self, local_state_dict, global_state_dict):
        vec_diff = vectorize_weight(local_state_dict) - vectorize_weight(global_state_dict)
        norm = torch.norm(vec_diff).item()
        clipped = vec_diff / max(1.0, norm / self.norm_bound)
        return load_model_weight_diff(local_state_dict, clipped, global_state_dict)

    def add_noise(self, local_weight: torch.Tensor, device=None, generator=None) -> torch.Tensor:
        noise = torch.randn(local_weight.size(), device=device or local_weight.device, generator=generator)
        return local_weight + noise * self.stddev

    # flat-arena variants (device hot path) -----------------------------------
    def clip_flat(self, local_rows: torch.Tensor, global_row: torch.Tensor, weight_mask=None) -> torch.Tensor:
        """Rows ``[n, P]`` of client params -> clipped in place around ``global_row``."""
        from ..ops import robust_clip_
        return robust_clip_(local_rows, global_row, self.norm_bound, weight_mask)

    def defend_slots_(self, upload: torch.Tensor, theta: torch.Tensor, n: torch.Tensor, weight_mask=None, seed: int = 0,
                      rnd: int = 0) -> torch.Tensor:
        """Apply the defense to a ``[C, M, P]`` upload arena in place before the cluster aggregation: every upload with
        ``n[c, m] > 0`` is clipped to distance ``norm_bound`` of its slot's model ``theta[m]`` (the model it trained from)
        and, for ``weak_dp``, gets ``stddev``-scaled ``gauss_hash`` noise of round ``rnd`` (``ops.reference.defense_seed``).
        Entries with ``weight_mask`` False (BatchNorm statistics) pass through.  Returns the update norms ``[C, M]``."""
        from ..ops import reference as ref, robust_clip_slots_
        std = self.stddev if self.defense_type == "weak_dp" else 0.0
        return robust_clip_slots_(upload, theta, n, self.norm_bound, weight_mask, std, ref.defense_seed(seed, rnd))


def make_defense(args) -> Optional[RobustAggregator]:
    """The robust-aggregation defense of the continual engines from ``args.defense_type`` (``none`` |
    ``norm_diff_clipping`` | ``weak_dp``), ``args.norm_bound`` (5.0) and ``args.stddev`` (0.025, weak_dp only); None for
    ``none``.  Raises ``ValueError`` for an unknown defense, a bound that is not finite or ≤ 0, or a negative stddev.

    ``weak_dp`` is the reference's backdoor defense (clipping plus Gaussian noise on each upload): it carries no (ε, δ)
    differential-privacy guarantee."""
    from ..ops.reference import defense_params
    name = str(getattr(args, "defense_type", "none") or "none")
    bound, _ = defense_params(name, getattr(args, "norm_bound", 5.0), getattr(args, "stddev", 0.025))
    if name == "none":
        return None
    ra = RobustAggregator(args)
    ra.defense_type, ra.norm_bound, ra.stddev = name, bound, float(getattr(args, "stddev", 0.025))
    return ra
