"""Record the reference's per-round client sampling into tests/golden/client_sampling.json (read by
tests/test_participation.py).

Run from the repository root with the original FedDrift tree at $FDB_REFERENCE_SRC:

    FDB_REFERENCE_SRC=/path/to/FedDrift python tools/record_client_sampling.py

It installs the unmodified reference into baseline/_ref (baseline/install_reference.py) and calls the reference aggregator's
``FedAvgEnsAggregatorSoftCluster.client_sampling(round_idx, C, K)`` (which reseeds numpy's global RNG with the round index)
for every case and round, storing the clients in the order the reference returns them.
"""
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "client_sampling.json")
CASES = [(10, 3), (100, 10), (7, 9)]   # (client_num_in_total, client_num_per_round)
ROUNDS = 200


def main():
    sys.path.insert(0, ROOT)
    from baseline import install_reference
    if install_reference.main() != 0:
        raise SystemExit("could not install the reference")
    # the parity test module knows how to import the installed reference (shims, disabled wandb)
    spec = importlib.util.spec_from_file_location("reference_parity", os.path.join(ROOT, "tests", "test_reference_parity.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.reference_module()
    from fedml_api.distributed.fedavg_ens.FedAvgEnsAggregatorSoftCluster import FedAvgEnsAggregatorSoftCluster as Agg
    cases = []
    for C, K in CASES:
        rounds = [[int(c) for c in Agg.client_sampling(None, r, C, K)] for r in range(ROUNDS)]
        cases.append({"client_num_in_total": C, "client_num_per_round": K, "rounds": rounds})
    with open(OUT, "w") as fh:
        json.dump({"cases": cases}, fh, separators=(",", ":"))
        fh.write("\n")
    print("wrote", OUT)


if __name__ == "__main__":
    main()
