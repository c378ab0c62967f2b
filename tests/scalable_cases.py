"""Cases of tests/test_scalable_lifting.py and the compiled reference's results
for them (oracle/_ref/libtmc13_scalable.so, oracle/scalable.mk): shared with
tests/golden/make_scalable_golden.py, which records those results in
tests/golden/scalable_golden.npz for machines without the reference."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))

import pcc_attr_b200 as pb  # noqa: E402
from pcc_attr_b200.synth import cloud_lidar, cloud_shell  # noqa: E402
from pcc_testlib import _pp, _ptr, make_lod_params, make_qpset  # noqa: E402

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libtmc13_scalable.so")


def lod_params(bias=(1, 1, 1), k=3, skip_layers=None, distribution=1):
    """lifting LoD fields (num_detail_levels and dist2 are not read with scalable
    lifting); intra-LoD prediction skipped at every level unless skip_layers"""
    lp = make_lod_params(levels=pb.SCALABLE_LODS, k=k, bias=bias, distribution=distribution,
                         skip_layers=skip_layers)
    return pb.LodParams.from_buffer_copy(bytes(lp))


def qpset():
    return pb.QpSet.from_buffer_copy(bytes(make_qpset(qp=34, chroma_offset=-2,
                                                      fixed_point_qp_offset=24)))


def _dense(n=6000, seed=3):
    return cloud_shell(n, bits=10, seed=seed)[0]


def _sparse(n=6000, seed=2):
    return cloud_lidar(n, seed=seed)[0]


def _partial(m, n=6000):
    """the points of a geometry decode stopped at octree level m: one per occupied
    node of size 2^m; geom_num_points counts the whole cloud"""
    full = _dense(n)
    xyz = np.unique((full >> m) << m, axis=0)
    return np.ascontiguousarray(xyz, dtype=np.int32), full.shape[0]


# name -> (lod params kwargs, max_neigh_range, min_geom_node_size_log2, cloud, geom_num_points)
def _lod_table():
    t = {
        "dense": ({}, 6, 0, lambda: _dense(), 0),
        "dense_bias118": (dict(bias=(1, 1, 8)), 6, 0, lambda: _dense(), 0),
        "dense_range1": ({}, 1, 0, lambda: _dense(), 0),
        "dense_range1_bias118": (dict(bias=(1, 1, 8)), 1, 0, lambda: _dense(), 0),
        "dense_intra_k2": (dict(skip_layers=0, k=2, distribution=0), 6, 0, lambda: _dense(), 0),
        "sparse_ring": ({}, 6, 0, lambda: _sparse(), 0),
        "sparse_ring_bias118": (dict(bias=(1, 1, 8)), 1, 0, lambda: _sparse(), 0),
        "duplicates": ({}, 6, 0, lambda: cloud_shell(3000, bits=8, seed=4, dups=True)[0], 0),
        "n1": ({}, 6, 0, lambda: _dense()[:1], 0),
        "n2": ({}, 6, 0, lambda: _dense()[:2], 0),
    }
    # partial1: geom_num_points = the whole cloud; partial2 / partial3: a slice
    # eight times larger (the skipped points outnumber the first level)
    for m, times in ((1, 1), (2, 8), (3, 8)):
        t[f"partial{m}"] = ({}, 6, m, (lambda m=m: _partial(m)[0]), (m, times))
    return t


LOD_CASES = list(_lod_table())
STOPS_AT_FIRST = ["partial2", "partial3"]
CONCATENATES_SEVERAL = ["sparse_ring", "partial1"]


def lod_case(name):
    kw, rng, m, cloud, geom = _lod_table()[name]
    xyz = np.ascontiguousarray(cloud(), dtype=np.int32)
    if geom:
        geom = _partial(geom[0])[1] * geom[1]
    return lod_params(**kw), pb.LodScalable(rng, m, geom, 0), xyz


def concatenated_levels(npl, n, scal):
    """levels at which buildPredictorsFast searched the earlier levels again
    (PCCTMC3Common.h:2377-2406), from numPointsInLod"""
    sizes = [int(x) for x in np.asarray(npl)[::-1]]  # build order: n, then retained counts
    skipped = scal.geom_num_points - n if scal.geom_num_points else 0
    on, count = True, 0
    for r, size in enumerate(sizes):
        refined = size - (sizes[r + 1] if r + 1 < len(sizes) else 0)
        start = n - size
        if not on or refined == 0:
            continue
        if refined <= start + skipped:
            on = False
        elif start > 0:
            count += 1
    return count


# lifting cases: name -> (cloud, max_neigh_range, lod params kwargs)
LIFT_CASES = ["dense", "sparse_ring", "dense_bias118"]


def lift_case(name, a):
    kw, rng, _, cloud, _ = _lod_table()[name]
    xyz = np.ascontiguousarray(cloud(), dtype=np.int32)
    if name == "sparse_ring":
        attrs = cloud_lidar(xyz.shape[0], seed=2, a=a)[1]
    else:
        attrs = cloud_shell(xyz.shape[0], bits=10, seed=3, a=a)[1]
    return lod_params(**kw), rng, xyz, np.ascontiguousarray(attrs, dtype=np.int32).reshape(len(xyz), a)


PARTIAL_CASES = ["partial1", "partial2", "partial3"]


def partial_case(name, a):
    """decoder inputs of a partial decode: levels of detail from the partial
    cloud, arbitrary quantised values and LCP coefficients"""
    lp, scal, xyz = lod_case(name)
    rng = np.random.default_rng(100 + scal.min_geom_node_size_log2 + a)
    values = rng.integers(-6, 7, size=(xyz.shape[0], a)).astype(np.int32)
    values[rng.random(xyz.shape[0]) < 0.5] = 0
    lcp = rng.integers(-2, 3, size=pb.SCALABLE_LODS).astype(np.int8) if a == 3 else None
    return lp, scal, xyz, values, lcp


# --------------------------------------------------------------------------
# the compiled reference

_ref = None


def _lib():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_LIB)
    return _ref


def ref_lod(lp, scal, xyz):
    n = xyz.shape[0]
    preds = np.zeros(n, dtype=pb.PREDICTOR_DTYPE)
    indexes = np.zeros(n, dtype=np.uint32)
    npl = np.zeros(pb.MAX_LODS, dtype=np.uint32)
    cnt = C.c_int32(0)
    _lib().tmc13ref_scalable_lod_build(
        C.byref(lp), C.c_int(scal.max_neigh_range), C.c_int(scal.min_geom_node_size_log2),
        C.c_int(scal.geom_num_points or n), _ptr(xyz, C.c_int32), C.c_int(n), _pp(preds),
        _ptr(indexes, C.c_uint32), _ptr(npl, C.c_uint32), C.byref(cnt))
    return preds, indexes, npl[:cnt.value].copy()


def ref_encode(lp, rng, xyz, attrs):
    n, a = attrs.shape
    values = np.zeros((n, a), dtype=np.int32)
    recon = np.zeros((n, a), dtype=np.int32)
    lcp = np.zeros(pb.SCALABLE_LODS, dtype=np.int8)
    q = qpset()
    _lib().tmc13ref_scalable_lift_encode(
        C.byref(lp), C.c_int(rng), C.byref(q), C.c_int(int(a == 3)), _ptr(xyz, C.c_int32),
        _ptr(attrs, C.c_int32), C.c_int(n), C.c_int(a), C.c_int(8), _ptr(values, C.c_int32),
        _ptr(recon, C.c_int32), _ptr(lcp, C.c_int8))
    return values, recon, lcp


def ref_partial_decode(name, a):
    lp, scal, xyz, values, lcp = partial_case(name, a)
    n = xyz.shape[0]
    cap = 64 + 16 * values.size
    buf = np.zeros(cap, dtype=np.uint8)
    length = _lib().tmc13ref_scalable_payload(_ptr(values, C.c_int32), C.c_int(n), C.c_int(a),
                                              _ptr(buf, C.c_uint8), C.c_int(cap))
    assert length > 0
    recon = np.zeros((n, a), dtype=np.int32)
    row = np.zeros(pb.SCALABLE_LODS, dtype=np.int8) if lcp is None else lcp
    q = qpset()
    _lib().tmc13ref_scalable_lift_decode(
        C.byref(lp), C.c_int(scal.max_neigh_range), C.c_int(scal.min_geom_node_size_log2),
        C.c_int(scal.geom_num_points), C.byref(q), C.c_int(int(a == 3)), _ptr(row, C.c_int8),
        _ptr(xyz, C.c_int32), C.c_int(n), C.c_int(a), C.c_int(8), _ptr(buf, C.c_uint8),
        C.c_int(length), _ptr(recon, C.c_int32))
    return recon


def million_point_slice():
    return np.ascontiguousarray(cloud_lidar(1000000, seed=2)[0], dtype=np.int32)
