"""Records the compiled reference's results for tests/test_recolour_exact.py
(nanoflann's trees and k-nearest lists, std::sort orders, recolourColour /
recolourReflectance) as SHA-256 digests (pcc_testlib.results_digest) into
tests/golden/recolour_exact_golden.npz.  Needs the reference libraries:
make -C oracle recolourref and make -C oracle -f recolour_codec.mk kdtreeref.

    python tests/golden/make_recolour_exact_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))

import test_recolour_exact as t  # noqa: E402
from pcc_testlib import results_digest  # noqa: E402


def main():
    assert t.live(), "the reference libraries under oracle/_ref are not built"
    entries = t.golden_entries()
    keys = sorted(entries)
    digests = np.stack([results_digest(entries[k]()) for k in keys])
    np.savez_compressed(t.GOLDEN, keys=np.array(keys), digests=digests)
    print(f"{len(keys)} digests -> {t.GOLDEN}")


if __name__ == "__main__":
    main()
