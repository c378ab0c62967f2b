"""CPU tests of the predicting-transform decoder: the product's bodies run on
the host (tests/emu/emu_pred.cpp) against the plain-C restatement of the
reference's decode loop (oracle/pred_oracle.c), in coding order and in random
orders of attempts that a dataflow launch may take; and the counter-driven
quantisation weights against the sequential walk."""
import ctypes as C

import numpy as np
import pytest

import pcc_attr_b200 as pb
from pcc_testlib import _pp, _ptr, synth_predictors
from pred_cases import GRID, load_emu_pred, make_case, oracle_pred_decode


def emu_decode(c):
    n, a = c["values"].shape
    out = np.zeros((n, a), dtype=np.int32)
    npl = np.ascontiguousarray(c["npl"], dtype=np.uint32)
    rc = load_emu_pred().emu_pred_decode(
        _pp(c["preds"]), _ptr(c["idx"], C.c_uint32), C.c_int(n), _ptr(npl, C.c_uint32),
        C.c_int(len(npl)), C.byref(c["qs"]), C.byref(c["pp"]), _ptr(c["qnw"], C.c_int32),
        _ptr(c["qpo"], C.c_int32), _ptr(c["icp"], C.c_int8), _ptr(c["values"], C.c_int32),
        C.c_int(a), C.c_int(c["bitdepth"]), _ptr(out, C.c_int32))
    return rc, out


def flow_weights(preds, npl, qnw, seed):
    qw = np.zeros(len(preds), dtype=np.uint64)
    npl = np.ascontiguousarray(npl, dtype=np.uint32)
    qnw = np.ascontiguousarray(qnw, dtype=np.int32)
    r = load_emu_pred().emu_quant_weights_flow(_pp(preds), C.c_int(len(preds)), _ptr(npl, C.c_uint32),
                                               C.c_int(len(npl)), _ptr(qnw, C.c_int32),
                                               C.c_uint(seed), _ptr(qw, C.c_uint64))
    return r, qw


def seq_weights(preds, npl, qnw):
    qw = np.zeros(len(preds), dtype=np.uint64)
    npl = np.ascontiguousarray(npl, dtype=np.uint32)
    qnw = np.ascontiguousarray(qnw, dtype=np.int32)
    rc = load_emu_pred().emu_quant_weights_fixed(_pp(preds), C.c_int(len(preds)), _ptr(npl, C.c_uint32),
                                                 C.c_int(len(npl)), _ptr(qnw, C.c_int32),
                                                 _ptr(qw, C.c_uint64))
    assert rc == 0
    return qw


def oracle_weights(preds, qnw):
    from pcc_testlib import load_oracle

    qw = np.zeros(len(preds), dtype=np.uint64)
    qnw = np.ascontiguousarray(qnw, dtype=np.int32)
    load_oracle().oracle_quant_weights_fixed(_pp(preds), C.c_int(len(preds)), _ptr(qnw, C.c_int32),
                                             _ptr(qw, C.c_uint64))
    return qw


@pytest.mark.parametrize("name,kw", GRID, ids=[g[0] for g in GRID])
def test_emu_pipeline_matches_oracle(name, kw):
    c = make_case(**kw)
    rc, out = emu_decode(c)
    assert rc == 0
    exp = oracle_pred_decode(c)
    assert np.array_equal(out, exp)
    # the case decodes to more than a constant
    assert c["values"].shape[0] < 3 or len(np.unique(exp)) > 1


@pytest.mark.parametrize("name,kw", [g for g in GRID if g[0].startswith(("cat", "skipall", "layers"))],
                         ids=lambda v: v if isinstance(v, str) else "")
def test_emu_dataflow_order_matches_oracle(name, kw):
    """PredDecodeFn attempted in random orders: refused attempts change
    nothing, and the result is the coding-order one"""
    c = make_case(**kw)
    n, a = c["values"].shape
    qw = oracle_weights(c["preds"], c["qnw"])
    qpo_pred = None if c["qpo"] is None else np.ascontiguousarray(c["qpo"][c["idx"]])
    npl = np.ascontiguousarray(c["npl"], dtype=np.uint32)
    exp = oracle_pred_decode(c)
    for seed in (1, 2):
        out = np.zeros((n, a), dtype=np.int32)
        refused = load_emu_pred().emu_pred_decode_sched(
            _pp(c["preds"]), _ptr(qw, C.c_uint64), C.c_int(n), _ptr(npl, C.c_uint32),
            C.c_int(len(npl)), C.byref(c["qs"]), C.byref(c["pp"]), _ptr(qpo_pred, C.c_int32),
            _ptr(c["icp"], C.c_int8), _ptr(c["values"], C.c_int32), C.c_int(a),
            C.c_int(c["bitdepth"]), C.c_uint(seed), _ptr(out, C.c_int32))
        assert refused > 0            # the schedule did meet unpublished neighbours
        assert np.array_equal(out[np.argsort(c["idx"])], exp)


@pytest.mark.parametrize("levels,skip", [(1, 0), (12, 0), (12, 4), (12, 13)])
def test_counter_driven_weights(levels, skip):
    c = make_case(n=4000, levels=levels, skip=skip, seed=5)
    for qnw in ((16, 8, 4), (255, 1, 0), (4, 4, 4)):
        exp = oracle_weights(c["preds"], qnw)
        assert np.array_equal(seq_weights(c["preds"], c["npl"], qnw), exp)
        r, qw = flow_weights(c["preds"], c["npl"], qnw, seed=levels + skip)
        assert r >= 0
        assert np.array_equal(qw, exp)


def test_counter_driven_weights_synthetic_chain():
    """a single level whose predictors reference the previous few points: the
    longest dependency chains"""
    n = 5000
    rng = np.random.default_rng(9)
    preds = np.zeros(n, dtype=pb.PREDICTOR_DTYPE)
    for i in range(1, n):
        k = min(3, i)
        preds["neighbor_count"][i] = k
        preds["predictor_index"][i, :k] = i - 1 - rng.integers(0, min(i, 4), size=k)
    npl = np.array([n], dtype=np.uint32)
    exp = oracle_weights(preds, (16, 8, 4))
    r, qw = flow_weights(preds, npl, (16, 8, 4), seed=3)
    assert r > 0
    assert np.array_equal(qw, exp)
    assert np.array_equal(seq_weights(preds, npl, (16, 8, 4)), exp)


def test_forward_reference_refused_on_host():
    c = make_case(n=500, levels=1, skip=0)
    preds = c["preds"].copy()
    i = int(np.nonzero(preds["neighbor_count"] > 0)[0][5])
    preds["predictor_index"][i, 0] = i + 3
    c["preds"] = preds
    rc, _ = emu_decode(c)
    assert rc == 1  # PCCB200_ERR_INVALID_ARG


def test_lifting_weights_unchanged_on_synthetic_lods():
    """the lifting-weight path keeps its inter-LoD form"""
    preds, npl = synth_predictors(3000, 6, seed=4)
    assert np.array_equal(seq_weights(preds, npl, (16, 8, 4)), oracle_weights(preds, (16, 8, 4)))


def test_pred_symbols_exported():
    import re
    import os
    from pcc_testlib import ROOT

    hdr = open(os.path.join(ROOT, "include", "pcc_attr_b200.h")).read()
    for name in ("pccb200_attr_pred_decode_lod", "pccb200_attr_pred_decode_multi_batch",
                 "pccb200_attr_pred_decode_multi_batch_dev"):
        assert re.search(r"\b" + name + r"\s*\(", hdr)
        assert name in pb.EXPORTS
        assert hasattr(pb.lib(), name)
    assert C.sizeof(pb.PredParams) == 16
