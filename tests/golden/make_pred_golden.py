"""Records the compiled reference's predicting-transform results for the cases
of tests/pred_cases.py REF_GRID (encoder payload decoded back to values, the
encoder's reconstruction, the decoder body's output, the reference's levels of
detail and ICP coefficients) in pred_golden.npz.  Needs oracle/_ref built by
`make -C oracle -f pred_codec.mk predref`."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "mpeg-pcc-tmc13_b200")]

from pred_cases import GOLDEN, GOLDEN_FIELDS, REF_GRID, ref_pred_case  # noqa: E402


def main():
    out = {}
    for nk in REF_GRID:
        c = ref_pred_case(nk)
        assert np.array_equal(c["recon"], c["ref_out"]), nk[0]
        for f in GOLDEN_FIELDS:
            if c[f] is None:
                continue
            v = c[f]
            out[f"{nk[0]}/{f}"] = v.view(np.uint8) if f == "preds" else v
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()
