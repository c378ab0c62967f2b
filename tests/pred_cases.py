"""Cases of the predicting-transform decoder tests: levels of detail of a
cloud, the APS fields of the transform, and values in coding order as the
reference's entropy decoding hands them to its loop (the prediction mode in
the low bits of the values)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import pcc_attr_b200 as pb
from pcc_testlib import (ROOT, _pp, _ptr, cloud_shell, load_oracle, make_lod_params, make_qpset,
                         oracle_lod_build)


def pred_params(max_direct=3, avg_disabled=0, threshold=64, icp=0):
    p = pb.PredParams()
    p.max_num_direct_predictors = max_direct
    p.direct_avg_predictor_disabled = avg_disabled
    p.adaptive_prediction_threshold = threshold
    p.icp_enabled = icp
    return p


def lod_params(levels=12, skip=0, decimation=0, blending=0):
    """the predicting transform's levels of detail: intra-LoD prediction on
    from level `skip` (levels + 1: off), like cfg/octree-predt-ctc-*"""
    p = make_lod_params(levels=levels, decimation=decimation, skip_layers=skip, blending=blending,
                        intra_range=0 if skip > levels else 1100000)
    return pb.LodParams.from_buffer_copy(bytes(p))


def cloud(n, seed, dup=False):
    xyz, _ = cloud_shell(n, bits=8 if n <= 100000 else 11, seed=seed)
    xyz = np.ascontiguousarray(xyz[:n], dtype=np.int32)
    if dup and n > 4:
        xyz[n // 2:n // 2 + n // 8] = xyz[:n // 8]   # duplicate points
    return xyz


def coding_values(n, a, bitdepth, seed, zeros=0.3):
    """values as the entropy decoder yields them: runs of zeros, small residuals
    with a mode in their low bits, and a few large ones"""
    rng = np.random.default_rng(seed)
    scale = 1 << max(0, bitdepth - 8)
    v = rng.integers(-24, 25, size=(n, a)) * rng.integers(1, 2 * scale + 1, size=(n, 1))
    big = rng.random(n) < 0.02
    v[big] = rng.integers(-(1 << bitdepth), 1 << bitdepth, size=(int(big.sum()), a))
    v[rng.random(n) < zeros] = 0
    return np.ascontiguousarray(v, dtype=np.int32)


def region_qpo(xyz, seed):
    """a qp-offset region: points of one octant get (d0, d1)"""
    rng = np.random.default_rng(seed)
    mid = np.median(xyz, axis=0)
    inside = np.all(xyz < mid, axis=1)
    qpo = np.zeros((xyz.shape[0], 2), dtype=np.int32)
    qpo[inside] = rng.integers(-6, 7, size=2)
    return qpo


def icp_rows(levels, seed):
    rng = np.random.default_rng(seed)
    r = rng.integers(-8, 9, size=(pb.MAX_LODS, 3)).astype(np.int8)
    r[:, 0] = 0
    return r


def make_case(n=3000, a=3, bitdepth=8, levels=12, skip=0, decimation=0, blending=0, max_direct=3,
              avg_disabled=0, threshold=64, icp=0, layers=None, qpo=False, dup=False, seed=1,
              qnw=(16, 8, 4), qp=10):
    """-> dict: lod params, xyz, the oracle's levels of detail, pred params,
    qpset, values, qpo, icp row"""
    xyz = cloud(n, seed, dup)
    lp = lod_params(levels, skip, decimation, blending)
    preds, idx, npl = oracle_lod_build(lp, xyz)
    return dict(lod=lp, xyz=xyz, preds=preds, idx=idx, npl=npl, levels=levels,
                pp=pred_params(max_direct, avg_disabled, threshold, icp),
                qs=pb.QpSet.from_buffer_copy(bytes(make_qpset(qp=qp, chroma_offset=2,
                                                              bitdepth=bitdepth, layers=layers))),
                values=coding_values(xyz.shape[0], a, bitdepth, seed + 7),
                qpo=region_qpo(xyz, seed) if qpo else None,
                icp=icp_rows(levels, seed) if (icp and a == 3) else None,
                a=a, bitdepth=bitdepth, qnw=np.array(qnw, dtype=np.int32))


def oracle_pred_decode(c, preds=None, idx=None, npl=None):
    """the plain-C restatement of the reference's decode loop -> [n, A] point order"""
    lib = load_oracle()
    preds = c["preds"] if preds is None else preds
    idx = c["idx"] if idx is None else idx
    npl = np.ascontiguousarray(c["npl"] if npl is None else npl, dtype=np.uint32)
    n, a = c["values"].shape
    out = np.zeros((n, a), dtype=np.int32)
    lib.oracle_pred_decode.restype = C.c_int
    rc = lib.oracle_pred_decode(
        _pp(preds), _ptr(idx, C.c_uint32), C.c_int(n), _ptr(npl, C.c_uint32), C.c_int(len(npl)),
        C.byref(c["qs"]), C.byref(c["pp"]), _ptr(c["qnw"], C.c_int32), _ptr(c["qpo"], C.c_int32),
        _ptr(c["icp"], C.c_int8), _ptr(c["values"], C.c_int32), C.c_int(a),
        C.c_int(c["bitdepth"]), _ptr(out, C.c_int32))
    assert rc == 0
    return out


# the grid of the GPU and host comparisons: (name, make_case kwargs)
GRID = [
    ("cat1_rgb_icp_blend", dict(a=3, icp=1, blending=1)),
    ("cat1_refl", dict(a=1)),
    ("rgb10", dict(a=3, bitdepth=10, icp=1)),
    ("refl16", dict(a=1, bitdepth=16)),
    ("rgb16", dict(a=3, bitdepth=16, threshold=0)),
    ("cat3_rgb", dict(a=3, levels=1, skip=0, avg_disabled=1, icp=1)),
    ("cat3_refl", dict(a=1, levels=1, skip=0, avg_disabled=1)),
    ("skipall_rgb", dict(a=3, skip=13)),
    ("skipall_refl", dict(a=1, skip=13, threshold=0)),
    ("dec1_rgb", dict(a=3, decimation=1)),
    ("dec2_refl", dict(a=1, decimation=2, blending=1)),
    ("layers_qpo_rgb", dict(a=3, layers=[(10, 2), (16, -2), (22, 1)], qpo=True, icp=1)),
    ("layers_qpo_refl", dict(a=1, layers=[(4, 0), (28, 0)], qpo=True)),
    ("dup_rgb", dict(a=3, dup=True, threshold=0)),
    ("qp40_refl", dict(a=1, qp=40, threshold=0)),
    ("n1_rgb", dict(n=1, a=3)),
    ("n2_refl", dict(n=2, a=1)),
] + [
    (f"mode_{a}_{md}_{ad}", dict(a=a, max_direct=md, avg_disabled=ad, threshold=t, seed=3 + md))
    for a in (1, 3) for md in range(4) for ad in (0, 1) for t in ((0,) if md % 2 else (64,))
]


_emu = None


def load_emu_pred():
    """tests/emu/emu_pred.cpp built for the host into a temporary directory"""
    global _emu
    if _emu is None:
        out = os.path.join(tempfile.mkdtemp(prefix="emu_pred_"), "libemu_pred.so")
        csrc = os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "csrc")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall",
                               "-Wno-unused-variable", "-x", "c++", "-I" + csrc,
                               "-I" + os.path.join(ROOT, "include"),
                               "-I" + os.path.join(ROOT, "tests", "emu"),
                               os.path.join(ROOT, "tests", "emu", "emu_pred.cpp"), "-o", out])
        _emu = C.CDLL(out)
        _emu.emu_pred_decode.restype = C.c_int
        _emu.emu_pred_decode_sched.restype = C.c_int64
        _emu.emu_quant_weights_flow.restype = C.c_int64
        _emu.emu_quant_weights_fixed.restype = C.c_int
    return _emu


# --------------------------------------------------------------------------
# the compiled reference (oracle/pred_codec.mk: _ref/libtmc13_pred.so)

REF_PRED = os.path.join(ROOT, "oracle", "_ref", "libtmc13_pred.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "pred_golden.npz")

# reference cases: (name, make_case kwargs); the attributes are a textured shell
REF_GRID = [
    ("cat1_rgb", dict(a=3, icp=1, blending=1, qp=10)),
    ("cat1_refl", dict(a=1, qp=10)),
    ("cat1_rgb_lossless", dict(a=3, icp=1, qp=4)),
    ("cat3_rgb", dict(a=3, levels=1, skip=0, avg_disabled=1, icp=1, qp=10)),
    ("cat3_refl", dict(a=1, levels=1, skip=0, avg_disabled=1, qp=4)),
    ("skipall_rgb", dict(a=3, skip=13, threshold=0, qp=16)),
    ("rgb10", dict(a=3, bitdepth=10, icp=1, qp=22, threshold=16)),
    ("refl16", dict(a=1, bitdepth=16, qp=40, threshold=8)),
    ("dec1_rgb", dict(a=3, decimation=1, qp=10)),
    ("dec2_refl", dict(a=1, decimation=2, blending=1, qp=10)),
    ("layers_rgb", dict(a=3, layers=[(10, 2), (16, -2), (22, 1)], icp=1)),
    ("n2_refl", dict(n=2, a=1)),
] + [
    (f"mode_{a}_{md}_{ad}", dict(a=a, max_direct=md, avg_disabled=ad, threshold=(md * 8) % 24,
                                 seed=3 + md, qp=10))
    for a in (1, 3) for md in range(4) for ad in (0, 1)
]
REF_GRID = [(nm, dict(dict(n=1500), **kw)) for nm, kw in REF_GRID]


def ref_pred_available():
    return os.path.exists(REF_PRED)


def attributes(xyz, a, bitdepth, seed):
    """a smooth field over the positions plus texture, so that neighbours
    differ by more or less than the thresholds"""
    rng = np.random.default_rng(seed)
    x = xyz.astype(np.float64)
    f = np.stack([np.sin(x[:, 0] / 17 + k) * np.cos(x[:, 1] / 23 - k) + x[:, 2] / 300 for k in range(a)], 1)
    top = (1 << bitdepth) - 1
    v = (f - f.min()) / (np.ptp(f) + 1e-9) * top * 0.8 + rng.normal(0, top * 0.04, size=f.shape)
    return np.ascontiguousarray(np.clip(np.rint(v), 0, top), dtype=np.int32)


def ref_pred_case(name_kw):
    """the reference's encoder and decoder bodies on one case -> dict of
    make_case fields with the reference's levels of detail, values (coding
    order), ICP coefficients, the encoder's reconstruction (recon) and the
    decoder body's output (ref_out)"""
    _, kw = name_kw
    c = make_case(**kw)
    lib = C.CDLL(REF_PRED)
    lib.tmc13ref_pred_encode.restype = C.c_int
    lib.tmc13ref_pred_decode.restype = C.c_int
    xyz = c["xyz"]
    n, a = xyz.shape[0], c["a"]
    attrs = attributes(xyz, a, c["bitdepth"], kw.get("seed", 1))
    buf = np.zeros(64 * n * a + 4096, dtype=np.uint8)
    recon = np.zeros((n, a), dtype=np.int32)
    preds = np.zeros(n, dtype=pb.PREDICTOR_DTYPE)
    idx = np.zeros(n, dtype=np.uint32)
    npl = np.zeros(pb.MAX_LODS, dtype=np.uint32)
    cnt = C.c_int32(0)
    icp = np.zeros((pb.MAX_LODS, 3), dtype=np.int8)
    ln = lib.tmc13ref_pred_encode(
        C.byref(c["lod"]), C.byref(c["qs"]), C.byref(c["pp"]), _ptr(c["qnw"], C.c_int32),
        _ptr(xyz, C.c_int32), _ptr(attrs, C.c_int32), C.c_int(n), C.c_int(a),
        C.c_int(c["bitdepth"]), _ptr(buf, C.c_uint8), C.c_int(buf.size), _ptr(recon, C.c_int32),
        _pp(preds), _ptr(idx, C.c_uint32), _ptr(npl, C.c_uint32), C.byref(cnt), _ptr(icp, C.c_int8))
    assert ln > 0, ln
    values = np.zeros((n, a), dtype=np.int32)
    out = np.zeros((n, a), dtype=np.int32)
    rc = lib.tmc13ref_pred_decode(
        C.byref(c["lod"]), C.byref(c["qs"]), C.byref(c["pp"]), _ptr(c["qnw"], C.c_int32),
        _ptr(xyz, C.c_int32), C.c_int(n), C.c_int(a), C.c_int(c["bitdepth"]), _ptr(buf, C.c_uint8),
        C.c_int(ln), _ptr(icp, C.c_int8), _ptr(values, C.c_int32), _ptr(out, C.c_int32))
    assert rc == 0
    c.update(preds=preds, idx=idx, npl=npl[:cnt.value].copy(), values=values,
             icp=icp if (a == 3 and kw.get("icp")) else None, recon=recon, ref_out=out)
    return c


# (positions come again from make_case; the reconstruction equals ref_out)
GOLDEN_FIELDS = ("preds", "idx", "npl", "values", "icp", "ref_out")


def golden_case(name_kw, g):
    """a REF_GRID case with the recorded reference results of pred_golden.npz"""
    name, kw = name_kw
    c = make_case(**kw)
    for f in GOLDEN_FIELDS:
        key = f"{name}/{f}"
        if key in g:
            v = g[key]
            c[f] = v.view(pb.PREDICTOR_DTYPE).reshape(-1) if f == "preds" else v
        elif f == "icp":
            c[f] = None
    return c
