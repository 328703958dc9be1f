"""Per-round client sampling (``--client_num_per_round``) of the device engine."""
from __future__ import annotations

import numpy as np


def sample_clients(round_idx: int, C: int, K: int) -> np.ndarray:
    """The ``min(K, C)`` clients that take part in round ``round_idx``, drawn without replacement.

    The same set as the reference's ``np.random.seed(round_idx); np.random.choice(range(C), K, replace=False)``
    (``FedAvgEnsAggregatorSoftCluster.client_sampling``), drawn from a private ``RandomState`` so numpy's global RNG is left
    alone.  The reference restarts ``round_idx`` at 0 every time step, so round r has the same participants at every step."""
    return np.random.RandomState(int(round_idx)).choice(range(C), min(int(K), int(C)), replace=False)
