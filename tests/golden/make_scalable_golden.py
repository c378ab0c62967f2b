"""Records the compiled reference's scalable-lifting results for the cases of
tests/scalable_cases.py in tests/golden/scalable_golden.npz (needs
oracle/_ref/libtmc13_scalable.so: `make -C oracle -f scalable.mk scalableref`).

    python tests/golden/make_scalable_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import scalable_cases as sc  # noqa: E402


def main():
    out = {}
    for name in sc.LOD_CASES:
        preds, indexes, npl = sc.ref_lod(*sc.lod_case(name))
        out[f"lod/{name}/preds"], out[f"lod/{name}/indexes"], out[f"lod/{name}/npl"] = preds, indexes, npl
    for name in sc.LIFT_CASES:
        for a in (3, 1):
            v, r, l = sc.ref_encode(*sc.lift_case(name, a))
            out[f"enc/{name}/{a}/values"], out[f"enc/{name}/{a}/recon"], out[f"enc/{name}/{a}/lcp"] = v, r, l
    for name in sc.PARTIAL_CASES:
        for a in (3, 1):
            out[f"dec/{name}/{a}/recon"] = sc.ref_partial_decode(name, a)
    np.savez_compressed(os.path.join(HERE, "scalable_golden.npz"), **out)


if __name__ == "__main__":
    main()
