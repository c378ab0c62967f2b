"""The predicting-transform decoder's oracle (oracle/pred_oracle.c) and the
product's host-emulated bodies against the compiled reference: its own
encode{Colors,Reflectances}Pred and decode{Colors,Reflectances}Pred bodies
(oracle/pred_codec.mk), live where the reference is built, and against the
recorded results of tests/golden/pred_golden.npz everywhere."""
import numpy as np
import pytest

from pred_cases import (GOLDEN, REF_GRID, golden_case, oracle_pred_decode, ref_pred_available,
                        ref_pred_case)
from test_pred_decode_host import emu_decode

IDS = [g[0] for g in REF_GRID]


@pytest.mark.skipif(not ref_pred_available(), reason="compiled reference not built")
@pytest.mark.parametrize("nk", REF_GRID, ids=IDS)
def test_oracle_equals_reference_live(nk):
    c = ref_pred_case(nk)
    # the decoder body reproduces the encoder's reconstruction from its own payload
    assert np.array_equal(c["ref_out"], c["recon"])
    assert np.array_equal(oracle_pred_decode(c), c["ref_out"])
    rc, out = emu_decode(c)
    assert rc == 0 and np.array_equal(out, c["ref_out"])


@pytest.mark.skipif(not ref_pred_available(), reason="compiled reference not built")
def test_goldens_are_the_live_reference():
    g = np.load(GOLDEN)
    for nk in REF_GRID[:6]:
        c = ref_pred_case(nk)
        gc = golden_case(nk, g)
        for f in ("values", "idx", "npl", "ref_out"):
            assert np.array_equal(gc[f], c[f]), (nk[0], f)
        assert np.array_equal(gc["preds"], c["preds"]), nk[0]


@pytest.mark.parametrize("nk", REF_GRID, ids=IDS)
def test_oracle_and_emulation_equal_goldens(nk):
    c = golden_case(nk, np.load(GOLDEN))
    assert np.array_equal(oracle_pred_decode(c), c["ref_out"])
    rc, out = emu_decode(c)
    assert rc == 0 and np.array_equal(out, c["ref_out"])
