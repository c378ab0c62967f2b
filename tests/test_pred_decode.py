"""GPU tests of the predicting-transform decoder (pccb200_attr_pred_decode_*):
bit-exact against the plain-C restatement of the reference's decode loop
(oracle/pred_oracle.c) over the grid of tests/pred_cases.py."""
import numpy as np
import pytest

import pcc_attr_b200 as pb
from pred_cases import GOLDEN, GRID, REF_GRID, golden_case, make_case, oracle_pred_decode

pytestmark = pytest.mark.gpu


def lod_decode(c, preds=None):
    h = pb.lod_import(c["preds"] if preds is None else preds, c["idx"], c["npl"], c["levels"])
    try:
        return pb.attr_pred_decode_lod(h, c["qs"], c["pp"], c["qnw"], c["values"],
                                       bitdepth=c["bitdepth"], qpoffs=c["qpo"], icp=c["icp"])
    finally:
        pb.lod_destroy(h)


@pytest.mark.parametrize("name,kw", GRID, ids=[g[0] for g in GRID])
def test_lod_entry_matches_oracle(name, kw):
    c = make_case(**kw)
    assert np.array_equal(lod_decode(c), oracle_pred_decode(c))


def _batch(cases, sets_per_unit=1):
    """units of one set each, or the same unit's values decoded as several
    sets: the call's arguments"""
    return dict(lods=[c["lod"] for c in cases], quant_neigh_weights=[c["qnw"] for c in cases],
                qpsets=[cases[0]["qs"]] * sets_per_unit, preds=[cases[0]["pp"]] * sets_per_unit,
                xyzs=[c["xyz"] for c in cases],
                values=[[c["values"]] * sets_per_unit for c in cases],
                bitdepths=[cases[0]["bitdepth"]] * sets_per_unit,
                qpoffs=[c["qpo"] for c in cases] if any(c["qpo"] is not None for c in cases) else None,
                icps=[[c["icp"]] * sets_per_unit for c in cases])


@pytest.mark.parametrize("name,kw", [g for g in GRID if not g[0].startswith("mode")],
                         ids=[g[0] for g in GRID if not g[0].startswith("mode")])
def test_batch_builds_lods_and_matches_oracle(name, kw):
    """the batch entry builds the levels of detail on the device"""
    c = make_case(**kw)
    out = pb.attr_pred_decode_multi_batch(**_batch([c]))
    assert np.array_equal(out[0][0], oracle_pred_decode(c))


@pytest.mark.parametrize("a", [1, 3])
def test_batch_of_units_matches_one_call_per_unit(a):
    kws = [dict(n=5000, a=a, seed=11), dict(n=1200, a=a, levels=1, skip=0, seed=12),
           dict(n=3000, a=a, skip=13, seed=13), dict(n=700, a=a, decimation=1, seed=14),
           dict(n=2, a=a, seed=15), dict(n=9000, a=a, levels=6, skip=2, seed=16, qpo=True)]
    cases = [make_case(**kw) for kw in kws] * 3          # 18 units
    # the same set parameters for every unit of the call
    for c in cases:
        c["qs"], c["pp"], c["bitdepth"] = cases[0]["qs"], cases[0]["pp"], cases[0]["bitdepth"]
        if c["qpo"] is None:
            c["qpo"] = np.zeros((c["xyz"].shape[0], 2), dtype=np.int32)
    out = pb.attr_pred_decode_multi_batch(**_batch(cases))
    for c, o in zip(cases, out):
        assert np.array_equal(o[0], oracle_pred_decode(c))
        one = pb.attr_pred_decode_multi_batch(**_batch([c]))
        assert np.array_equal(o[0], one[0][0])


def test_sets_share_the_levels_of_detail():
    c = make_case(n=6000, a=3, icp=1, seed=21)
    r = make_case(n=6000, a=1, seed=21, threshold=0)
    out = pb.attr_pred_decode_multi_batch(
        lods=[c["lod"]], quant_neigh_weights=[c["qnw"]], qpsets=[c["qs"], r["qs"]],
        preds=[c["pp"], r["pp"]], xyzs=[c["xyz"]], values=[[c["values"], r["values"]]],
        bitdepths=[8, 8], icps=[[c["icp"], None]])
    assert np.array_equal(out[0][0], oracle_pred_decode(c))
    assert np.array_equal(out[0][1], oracle_pred_decode(r))


def test_dev_matches_host():
    torch = pytest.importorskip("torch")
    cases = [make_case(n=4000, a=3, icp=1, seed=31, qpo=True),
             make_case(n=2500, a=3, icp=1, seed=32, levels=1, skip=0, qpo=True)]
    cases[1]["qs"], cases[1]["pp"] = cases[0]["qs"], cases[0]["pp"]
    host = pb.attr_pred_decode_multi_batch(**_batch(cases))
    dx = [torch.from_numpy(c["xyz"]).cuda() for c in cases]
    dq = [torch.from_numpy(c["qpo"]).cuda() for c in cases]
    dv = [torch.from_numpy(c["values"]).cuda() for c in cases]
    do = [torch.zeros_like(v) for v in dv]
    torch.cuda.synchronize()
    pb.attr_pred_decode_multi_batch_dev(
        [c["lod"] for c in cases], [c["qnw"] for c in cases], [cases[0]["qs"]], [cases[0]["pp"]],
        [3], [x.data_ptr() for x in dx], [c["xyz"].shape[0] for c in cases],
        [[v.data_ptr()] for v in dv], [[o.data_ptr()] for o in do], bitdepths=[8],
        d_qpoffs=[q.data_ptr() for q in dq], icps=[[c["icp"]] for c in cases])
    torch.cuda.synchronize()
    for h, o in zip(host, do):
        assert np.array_equal(h[0], o.cpu().numpy())


def test_forward_reference_is_refused_before_decoding():
    c = make_case(n=2000, levels=1, skip=0, seed=41)
    preds = c["preds"].copy()
    i = int(np.nonzero(preds["neighbor_count"] > 0)[0][10])
    preds["predictor_index"][i, 0] = i + 5
    with pytest.raises(pb.PccB200Error, match="status 1"):
        lod_decode(c, preds)
    # the library keeps working
    assert np.array_equal(lod_decode(c), oracle_pred_decode(c))


def test_scalable_handle_unsupported():
    c = make_case(n=500, seed=42)
    scal = pb.LodScalable()
    scal.max_neigh_range = 1
    h = pb.lod_import(c["preds"], c["idx"], c["npl"], c["levels"], scal=scal)
    try:
        with pytest.raises(pb.PccB200Error, match="status 5"):
            pb.attr_pred_decode_lod(h, c["qs"], c["pp"], c["qnw"], c["values"])
    finally:
        pb.lod_destroy(h)


def test_quant_weights_fixed_1m_single_level():
    """a 1M-point level that references itself: the counter-driven dataflow"""
    from test_pred_decode_host import oracle_weights

    n = 1 << 20
    rng = np.random.default_rng(7)
    preds = np.zeros(n, dtype=pb.PREDICTOR_DTYPE)
    i = np.arange(n)
    cnt = np.minimum(3, i)
    preds["neighbor_count"] = cnt
    back = rng.integers(1, 40, size=(n, 3))
    idx = np.maximum(i[:, None] - back, 0)
    idx[cnt[:, None] <= np.arange(3)[None, :]] = 0
    preds["predictor_index"] = idx
    for qnw in ((16, 8, 4), (64, 32, 16)):
        qw = pb.quant_weights_fixed(preds, np.array([n], dtype=np.uint32), qnw)
        assert np.array_equal(qw, oracle_weights(preds, qnw))


@pytest.mark.parametrize("nk", REF_GRID, ids=[g[0] for g in REF_GRID])
def test_lod_and_batch_entries_equal_reference_goldens(nk):
    """the reference decoder body's recorded output: on its own levels of
    detail (imported), and on the levels of detail the batch entry builds"""
    c = golden_case(nk, np.load(GOLDEN))
    assert np.array_equal(lod_decode(c), c["ref_out"])
    out = pb.attr_pred_decode_multi_batch(**_batch([c]))
    assert np.array_equal(out[0][0], c["ref_out"])
