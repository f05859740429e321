"""Generates tests/golden/ref_digests.json FROM THE REFERENCE ITSELF:  python tests/golden/make_ref_digests.py [--new]

Runs every scenario of tests/ref_scenarios.py on oracle/_ref/libgg_ref.so (the reference's unmodified sources on CPU
stand-ins, built by oracle/build_ref.py from a checkout of the reference) and stores one digest per value the
reference answered with, and the reference's labels of one scan at thread_count = 1 (ref_labels_*.npz).
tests/test_oracle_vs_ref.py replays them on the oracle port and tests/test_gpu_parity.py on
the CUDA path.  With --new only the scenarios that have no stored digests yet are run and added; every stored entry and
the labels file stay as they are.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import ref_scenarios as rs  # noqa: E402
from oracle import ref as refmod  # noqa: E402


def main():
    if not refmod.available():
        raise SystemExit("oracle/_ref/libgg_ref.so is missing: build it with oracle/build_ref.py first")
    only_new = "--new" in sys.argv[1:]
    out = {}
    if only_new:
        with open(rs.DIGESTS) as f:
            out = json.load(f)
    for name, (_, arg_sets) in rs.SCENARIOS.items():
        for args in arg_sets:
            if rs.key(name, args) in out:
                continue
            out[rs.key(name, args)] = rs.run(name, rs.Reference, *args, record=True)
            print(rs.key(name, args), len(out[rs.key(name, args)]), "values", flush=True)
    with open(rs.DIGESTS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    if only_new:
        return
    dim, res, pts, org = rs.sequential_scan()
    r = refmod.Reference(dim, res)   # thread_count = 1
    r.init_map(0.0, 0.0, 0.0)
    np.savez_compressed(rs.SEQUENTIAL_LABELS, labels=r.filter_cloud(pts, org, 0.0)[0])


if __name__ == "__main__":
    main()
