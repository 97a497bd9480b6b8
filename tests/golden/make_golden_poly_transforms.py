"""Writes tests/golden/poly_transforms.json: the SHA-256 of the oracle's results (oracle_dense/capi.cpp orcd_poly_*) on
the seeded full-width inputs of tests/poly_transform_cases.py: k sequential top and bottom binds, split at len/2 and
len/8 at 2^22 and 2^24 evaluations, and new_padded of 2^22 + 1 evaluations.  The arrays hashed are the results'
evaluations as (n, 4) little-endian u64 Montgomery limbs, the layout lasso_poly_read returns."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import poly_transform_cases as pt  # noqa: E402


def main():
    cases = {}
    for nv in pt.GOLDEN_NV:
        Z, r = pt.golden_inputs(nv)
        for k in pt.GOLDEN_K:
            cases["top_nv%d_k%d" % (nv, k)] = pt.sha(pt.bind(Z, r[:k], True))
            cases["bot_nv%d_k%d" % (nv, k)] = pt.sha(pt.bind(Z, r[:k], False))
        for d in pt.SPLIT_DIV:
            lo, hi = pt.split(Z, Z.shape[0] // d)
            cases["split_nv%d_div%d" % (nv, d)] = [pt.sha(lo), pt.sha(hi)]
        print("nv", nv, "done", flush=True)
    cases["padded_%d" % pt.PADDED_LEN] = pt.sha(pt.new_padded(pt.padded_input()))
    json.dump({"generator": "tests/golden/make_golden_poly_transforms.py", "cases": cases},
              open(os.path.join(HERE, "poly_transforms.json"), "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
