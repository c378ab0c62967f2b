"""Levels of detail imported from the caller (pccb200_lod_import) and the
lifting drop-in (host/lift_dropin.cpp) that hands the reference's own _lods to
the library from inside AttributeEncoder / AttributeDecoder.

CPU: every malformed import argument is refused before a device is looked up,
and the drop-in's fallback to the reference's aliased bodies writes the
reference's bitstream.  GPU: coding on an imported handle equals the library's
own lifting entries bit for bit, bad imports are refused, and tmc3 with the
drop-in (oracle/lift_codec.mk) writes md5-identical bitstreams, encoder
reconstructions and decoder output against the unmodified tmc3."""
import ctypes as C
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

import pcc_attr_b200 as pb
import scalable_cases as sc
from pcc_testlib import ROOT, cloud_random, cloud_shell, make_lod_params, make_qpset
from pcc_attr_b200.synth import texture

INVALID_ARG = 1
UNSUPPORTED = 5
LIFT_BIN = os.path.join(ROOT, "oracle", "_ref", "tmc3_b200_lift")


def _import_rc(preds, idx, n, npl, lod_count, levels, scal=None, out=True):
    h = C.c_void_p()
    rc = pb.lib().pccb200_lod_import(
        None if preds is None else C.cast(preds.ctypes.data, C.POINTER(pb.Predictor)),
        None if idx is None else idx.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_int32(n),
        None if npl is None else npl.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_int32(lod_count),
        C.c_int32(levels), C.byref(scal) if scal is not None else None,
        C.byref(h) if out else None)
    if h.value:
        pb.lod_destroy(h.value)
    return rc


def _toy(n=8):
    preds = np.zeros(n, dtype=pb.PREDICTOR_DTYPE)
    idx = np.arange(n, dtype=np.uint32)
    npl = np.zeros(pb.MAX_LODS + 1, dtype=np.uint32)
    npl[:2] = (2, n)
    return preds, idx, npl


def test_import_malformed_arguments_need_no_device():
    """each malformed argument returns PCCB200_ERR_INVALID_ARG, not NO_DEVICE"""
    preds, idx, npl = _toy()
    S = pb.LodScalable
    assert _import_rc(None, idx, 8, npl, 2, 2) == INVALID_ARG
    assert _import_rc(preds, None, 8, npl, 2, 2) == INVALID_ARG
    assert _import_rc(preds, idx, 8, None, 2, 2) == INVALID_ARG
    assert _import_rc(preds, idx, 8, npl, 2, 2, out=False) == INVALID_ARG
    assert _import_rc(preds, idx, 0, npl, 2, 2) == INVALID_ARG
    assert _import_rc(preds, idx, 8, npl, 0, 2) == INVALID_ARG
    big = np.arange(1, pb.MAX_LODS + 2, dtype=np.uint32)
    big[-1] = 8 + pb.MAX_LODS
    assert _import_rc(np.zeros(8 + pb.MAX_LODS, dtype=pb.PREDICTOR_DTYPE),
                      np.arange(8 + pb.MAX_LODS, dtype=np.uint32), 8 + pb.MAX_LODS, big,
                      pb.MAX_LODS + 1, pb.MAX_LODS + 1) == INVALID_ARG  # more than MAX_LODS levels
    dec = npl.copy()
    dec[:3] = (5, 3, 8)
    assert _import_rc(preds, idx, 8, dec, 3, 3) == INVALID_ARG  # decreasing counts
    zero = npl.copy()
    zero[:2] = (0, 8)
    assert _import_rc(preds, idx, 8, zero, 2, 2) == INVALID_ARG  # first count 0
    assert _import_rc(preds, idx, 9, npl, 2, 2) == INVALID_ARG  # last count != n
    assert _import_rc(preds, idx, 8, npl, 2, 1) == INVALID_ARG  # num_detail_levels < lod_count
    assert _import_rc(preds, idx, 8, npl, 2, pb.MAX_LODS + 1) == INVALID_ARG
    assert _import_rc(preds, idx, 8, npl, 2, 2, S(1, 0, 0, 1)) == INVALID_ARG  # reserved
    assert _import_rc(preds, idx, 8, npl, 2, 2, S(1, 21, 0, 0)) == INVALID_ARG
    assert _import_rc(preds, idx, 8, npl, 2, 2, S(1, -1, 0, 0)) == INVALID_ARG
    assert _import_rc(preds, idx, 8, npl, 2, 2, S(1, 0, 7, 0)) == INVALID_ARG  # geom < n


def test_import_exported():
    assert "pccb200_lod_import" in pb.EXPORTS
    assert hasattr(pb.lib(), "pccb200_lod_import")


def _md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def _run(binary, args, strict):
    env = dict(os.environ)
    if strict:
        env["PCCB200_DROPIN_STRICT"] = "1"
    else:
        env.pop("PCCB200_DROPIN_STRICT", None)
    r = subprocess.run([binary] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       env=env)
    return r.returncode, r.stdout


def _encode_both(tmp_path, ply, flags, strict):
    import codec_harness as ch

    out = {}
    for name, binary in (("ref", ch.REF_BIN), ("lift", LIFT_BIN)):
        b, r = str(tmp_path / f"{name}.bin"), str(tmp_path / f"{name}_rec.ply")
        rc, log = _run(binary, [f"--uncompressedDataPath={ply}", f"--compressedStreamPath={b}",
                                f"--reconstructedDataPath={r}"] + flags, strict)
        assert rc == 0, log[-2000:]
        out[name] = (b, r, log)
    return out


def _decode_both(tmp_path, bitstream, strict, extra=()):
    import codec_harness as ch

    md5s = []
    for name, binary in (("ref", ch.REF_BIN), ("lift", LIFT_BIN)):
        d = str(tmp_path / f"d{name}.ply")
        rc, log = _run(binary, ["--mode=1", f"--compressedStreamPath={bitstream}",
                                f"--reconstructedDataPath={d}", "--convertPlyColourspace=0",
                                *extra], strict and name == "lift")
        if rc != 0 and name == "ref":
            return None, log
        assert rc == 0, log[-2000:]
        md5s.append(_md5(d))
    return md5s, ""


def _need_codec():
    import codec_harness as ch

    if not (os.path.exists(ch.REF_BIN) and os.path.exists(LIFT_BIN)):
        pytest.skip("oracle/_ref/tmc3_ref and tmc3_b200_lift not built (oracle/lift_codec.mk)")


def _write_ply(path, xyz, rgb, refl=None):
    with open(path, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
                % len(xyz))
        if refl is not None:
            f.write("property uint16 refc\n")
        f.write("end_header\n")
        for i in range(len(xyz)):
            row = "%d %d %d %d %d %d" % (*xyz[i], *rgb[i])
            f.write(row + (" %d\n" % refl[i] if refl is not None else "\n"))


def _lift_flags(decimator=0, lods=10, extra=(), refl=False):
    """cfg/octree-liftt-ctc-lossless-geom-lossy-attrs.yaml, colour (attribute
    options precede the --attribute they apply to); refl: then a 16-bit
    reflectance"""
    import codec_harness as ch

    f = [x for x in ch.lod_flags(34, 2, decimator=decimator, lods=lods)
         if not x.startswith(("--convertPlyColourspace", "--attribute"))]
    f += ["--convertPlyColourspace=0", *extra, "--attribute=color"]
    if refl:
        f += ["--bitdepth=16", *extra, "--attribute=reflectance"]
    return f


def test_fallback_path_matches_reference(tmp_path):
    """more levels of detail than the library takes: the drop-in runs the
    reference's aliased bodies (no device needed) and the bitstream, the
    encoder reconstruction and the decoder output match the unmodified tmc3;
    with PCCB200_DROPIN_STRICT=1 the same run fails instead"""
    _need_codec()
    xyz, rgb = cloud_shell(20000, bits=10, seed=12)
    ply = str(tmp_path / "in.ply")
    _write_ply(ply, xyz, texture(rgb, 20, 5))
    flags = _lift_flags(lods=40)
    out = _encode_both(tmp_path, ply, flags, strict=False)
    assert _md5(out["ref"][0]) == _md5(out["lift"][0]), "bitstreams differ"
    assert _md5(out["ref"][1]) == _md5(out["lift"][1]), "encoder reconstructions differ"
    md5s, _ = _decode_both(tmp_path, out["ref"][0], strict=False)
    assert md5s[0] == md5s[1]
    rc, log = _run(LIFT_BIN, [f"--uncompressedDataPath={ply}",
                              f"--compressedStreamPath={tmp_path / 's.bin'}",
                              f"--reconstructedDataPath={tmp_path / 's.ply'}"] + flags, True)
    assert rc != 0 and "lift drop-in" in log


# --------------------------------------------------------------------------
# GPU: the import against the library's own entries

# name: (cloud kind, make_lod_params kwargs)
LOD_CONFIGS = {
    "distance": ("shell", dict(levels=12)),
    "periodic": ("shell", dict(levels=12, decimation=1)),
    "centroid": ("random", dict(levels=12, decimation=2)),
    "one_level": ("shell", dict(levels=1)),
}


def _cloud(kind, n=20000, seed=11):
    if kind == "shell":
        xyz, rgb = cloud_shell(n, bits=9, seed=seed)
    else:
        xyz, rgb = cloud_random(n, 8, seed)
    return np.ascontiguousarray(xyz), np.ascontiguousarray(texture(rgb, 20, seed + 1).astype(np.int32))


def _refl(rgb, bits, seed=3):
    r = (rgb[:, :1].astype(np.int64) * 2 + rgb[:, 1:2]) // 3
    if bits == 16:
        rng = np.random.default_rng(seed)
        r = np.clip(r * 257 + rng.integers(-4000, 4001, size=r.shape), 0, 65535)
    return np.ascontiguousarray(r.astype(np.int32))


def _qpset(**kw):
    return pb.QpSet.from_buffer_copy(bytes(make_qpset(fixed_point_qp_offset=24, **kw)))


# name: (attribute set, lcp, bit depth, qpset kwargs, point qp offsets)
SETS = {
    "rgb_lcp": ("rgb", 1, 8, dict(qp=30, chroma_offset=-2), False),
    "rgb_nolcp": ("rgb", 0, 8, dict(qp=30, chroma_offset=-2), False),
    "refl8": ("refl", 0, 8, dict(qp=40, chroma_offset=0), False),
    "refl16": ("refl", 0, 16, dict(qp=40, chroma_offset=0, bitdepth=16), False),
    "rgb_qp_layers": ("rgb", 1, 8, dict(layers=[(28, -2), (34, 1), (40, 3)]), False),
    "rgb_point_qp": ("rgb", 1, 8, dict(qp=30, chroma_offset=-2), True),
    "refl_point_qp_layers": ("refl", 0, 8, dict(layers=[(36, 0), (44, 0)]), True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(LOD_CONFIGS))
@pytest.mark.parametrize("setname", list(SETS))
def test_gpu_import_equals_attr_lift(config, setname):
    kind, kw = LOD_CONFIGS[config]
    kind_set, lcp, bits, qkw, point_qp = SETS[setname]
    xyz, rgb = _cloud(kind)
    attrs = rgb if kind_set == "rgb" else _refl(rgb, bits)
    lp = pb.LodParams.from_buffer_copy(bytes(make_lod_params(**kw)))
    q = _qpset(**qkw)
    qpo = None
    if point_qp:
        rng = np.random.default_rng(7)
        qpo = rng.integers(-6, 7, size=(len(xyz), 2)).astype(np.int32)
        qpo[rng.random(len(xyz)) < 0.6] = 0
    ev, er, el = pb.attr_lift_encode(lp, q, xyz, attrs, lcp_enabled=lcp, bitdepth=bits, qpoffs=qpo)
    preds, idx, npl = pb.lod_build(lp, xyz)
    h = pb.lod_import(preds, idx, npl, lp.num_detail_levels)
    try:
        v, r, row = pb.attr_lift_encode_lod(h, q, attrs, lcp_enabled=lcp, bitdepth=bits, qpoffs=qpo)
        assert np.array_equal(v, ev) and np.array_equal(r, er)
        assert np.array_equal(row[:lp.num_detail_levels], el)
        lcp_in = el if lcp and attrs.shape[1] == 3 else None
        d = pb.attr_lift_decode_lod(h, q, v, lcp=lcp_in, bitdepth=bits, qpoffs=qpo)
        assert np.array_equal(d, pb.attr_lift_decode(lp, q, xyz, ev, lcp=lcp_in, bitdepth=bits,
                                                     qpoffs=qpo))
        assert np.array_equal(d, er)
        assert pb.lib().pccb200_lod_reusable(C.c_void_p(h), C.byref(lp)) == 0
    finally:
        pb.lod_destroy(h)


@pytest.mark.gpu
def test_gpu_scalable_import_equals_attr_lift_scalable():
    """scalable levels of detail imported with the encoder's (n, 0) weights,
    colour with LCP and reflectance; then partial decodes with the decoder's
    (geom_num_points, min_geom_node_size_log2) weights"""
    q = sc.qpset()
    for name in sc.LIFT_CASES:
        for a in (3, 1):
            lp, rng, xyz, attrs = sc.lift_case(name, a)
            scal = pb.LodScalable(rng, 0, 0, 0)
            vals, recs, lcps = pb.attr_lift_scalable(True, [lp], [scal], [q], [xyz], [[attrs]],
                                                     lcp_enabled=[int(a == 3)])
            preds, idx, npl = pb.lod_build_scalable(lp, scal, xyz)
            h = pb.lod_import(preds, idx, npl, pb.SCALABLE_LODS, pb.LodScalable(1, 0, len(xyz), 0))
            try:
                v, r, row = pb.attr_lift_encode_lod(h, q, attrs, lcp_enabled=int(a == 3))
                assert np.array_equal(v, vals[0][0]) and np.array_equal(r, recs[0][0])
                if a == 3:
                    assert np.array_equal(row[:pb.SCALABLE_LODS], lcps[0][0])
                d = pb.attr_lift_decode_lod(h, q, v, lcp=row[:pb.SCALABLE_LODS] if a == 3 else None)
                assert np.array_equal(d, r)
            finally:
                pb.lod_destroy(h)
    for name in sc.PARTIAL_CASES:
        for a in (3, 1):
            lp, scal, xyz, values, lcp = sc.partial_case(name, a)
            want = pb.attr_lift_scalable(False, [lp], [scal], [q], [xyz], [[values]],
                                         lcp_enabled=[int(a == 3)], lcps=[[lcp]])[0][0]
            preds, idx, npl = pb.lod_build_scalable(lp, scal, xyz)
            h = pb.lod_import(preds, idx, npl, pb.SCALABLE_LODS,
                              pb.LodScalable(1, scal.min_geom_node_size_log2, scal.geom_num_points, 0))
            try:
                got = pb.attr_lift_decode_lod(h, q, values, lcp=lcp if a == 3 else None)
            finally:
                pb.lod_destroy(h)
            assert np.array_equal(got, want)


@pytest.mark.gpu
def test_gpu_import_rejects_bad_levels():
    """a non-permutation and an out-of-range neighbour are refused by the
    import (on the device); an own-level reference by the lifting call"""
    xyz, rgb = _cloud("shell", n=5000)
    lp = pb.LodParams.from_buffer_copy(bytes(make_lod_params(levels=8)))
    preds, idx, npl = pb.lod_build(lp, xyz)
    n, cnt = len(xyz), len(npl)
    full = np.zeros(pb.MAX_LODS, dtype=np.uint32)
    full[:cnt] = npl
    dup = idx.copy()
    dup[0] = dup[1]
    assert _import_rc(preds, dup, n, full, cnt, 8) == INVALID_ARG
    out = idx.copy()
    out[3] = n
    assert _import_rc(preds, out, n, full, cnt, 8) == INVALID_ARG
    far = preds.copy()
    j = int(np.nonzero(far["neighbor_count"] > 0)[0][-1])
    far["predictor_index"][j, 0] = n
    assert _import_rc(far, idx, n, full, cnt, 8) == INVALID_ARG
    assert _import_rc(preds, idx, n, full, cnt, 8) == 0
    own = preds.copy()
    last = int(npl[-2])
    k = int(np.nonzero(own["neighbor_count"][last:] > 0)[0][0]) + last
    own["predictor_index"][k, 0] = last  # in its own (the last) level
    h = pb.lod_import(own, idx, npl, 8)
    try:
        attrs = np.ascontiguousarray(rgb)
        vals = np.zeros_like(attrs)
        row = np.zeros(pb.MAX_LODS, dtype=np.int8)
        rc = pb.lib().pccb200_attr_lift_encode_lod(
            C.c_void_p(h), C.byref(_qpset(qp=30, chroma_offset=-2)), C.c_int32(1), None,
            attrs.ctypes.data_as(C.POINTER(C.c_int32)), C.c_int32(3), C.c_int32(8),
            vals.ctypes.data_as(C.POINTER(C.c_int32)), row.ctypes.data_as(C.POINTER(C.c_int8)))
        assert rc == UNSUPPORTED
    finally:
        pb.lod_destroy(h)


# --------------------------------------------------------------------------
# GPU: the whole codec

# name: (encoder flags beyond the lifting CTC ones, colour + reflectance)
CODEC_CASES = {
    "decimator0": (dict(decimator=0), [], False),
    "decimator1": (dict(decimator=1), [], False),
    "decimator2": (dict(decimator=2), [], False),
    "lods1": (dict(lods=1), [], False),
    "lods12": (dict(lods=12), [], False),
    "qp_layers": (dict(), ["--qpLayerOffsetsLuma=0,3,-2", "--qpLayerOffsetsChroma=0,1,2"], False),
    "no_lcp": (dict(), ["--lastComponentPredictionEnabled=0"], False),
    "colour_refl16_slices": (dict(), [], True),
}


def _codec_input(tmp_path, refl):
    xyz, rgb = cloud_shell(40000, bits=10, seed=31)
    rgb = texture(rgb, 24, 32)
    r16 = None
    if refl:
        r16 = (rgb[:, 0].astype(np.int64) * 3 + rgb[:, 2]) * 61
    ply = str(tmp_path / "in.ply")
    _write_ply(ply, xyz, rgb, r16)
    return ply, xyz


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CODEC_CASES))
def test_whole_codec_lift(tmp_path, case):
    """tmc3 with the lifting drop-in (PCCB200_DROPIN_STRICT=1: no fallback)
    against the unmodified tmc3: bitstream, encoder reconstruction and the
    decoder output of the reference's bitstream md5-identical"""
    _need_codec()
    kw, extra, refl = CODEC_CASES[case]
    ply, _ = _codec_input(tmp_path, refl)
    flags = _lift_flags(**kw, extra=extra, refl=refl)
    if refl:
        flags = ["--partitionMethod=4", "--sliceMaxPoints=15000", "--sliceMinPoints=5000"] + flags
    out = _encode_both(tmp_path, ply, flags, strict=True)
    if case == "colour_refl16_slices":
        slices = re.search(r"Slice number: (\d+)", out["ref"][2])
        assert slices and int(slices.group(1)) > 1, "one slice only"
    assert _md5(out["ref"][0]) == _md5(out["lift"][0]), "bitstreams differ"
    assert _md5(out["ref"][1]) == _md5(out["lift"][1]), "encoder reconstructions differ"
    md5s, _ = _decode_both(tmp_path, out["ref"][0], strict=True)
    assert md5s[0] == md5s[1]


@pytest.mark.gpu
def test_whole_codec_lift_not_strict(tmp_path):
    """the same run without PCCB200_DROPIN_STRICT: nothing changes"""
    _need_codec()
    ply, _ = _codec_input(tmp_path, False)
    out = _encode_both(tmp_path, ply, _lift_flags(), strict=False)
    assert _md5(out["ref"][0]) == _md5(out["lift"][0])
    assert _md5(out["ref"][1]) == _md5(out["lift"][1])
    md5s, _ = _decode_both(tmp_path, out["ref"][0], strict=False)
    assert md5s[0] == md5s[1]


@pytest.mark.gpu
def test_whole_codec_lift_scalable(tmp_path):
    """scalable lifting, strict: full encode and decode, then a partial decode
    (--decodeMaxPoints, minGeomNodeSizeLog2 > 0) of the reference's bitstream"""
    _need_codec()
    xyz, rgb = cloud_shell(60000, bits=10, seed=12)
    ply = str(tmp_path / "in.ply")
    _write_ply(ply, xyz, rgb)
    flags = ["--positionQpMultiplierLog2=3", "--pointCountMetadata=1"] + _lift_flags(
        extra=["--aps_scalable_enable_flag=1"])
    out = _encode_both(tmp_path, ply, flags, strict=True)
    assert _md5(out["ref"][0]) == _md5(out["lift"][0]), "bitstreams differ"
    assert _md5(out["ref"][1]) == _md5(out["lift"][1]), "encoder reconstructions differ"
    md5s, _ = _decode_both(tmp_path, out["ref"][0], strict=True)
    assert md5s[0] == md5s[1]
    md5s, log = _decode_both(tmp_path, out["ref"][0], strict=True,
                             extra=[f"--decodeMaxPoints={xyz.shape[0] // 4}"])
    if md5s is None:
        pytest.skip("the reference decoder rejects --decodeMaxPoints on this stream: " + log[-300:])
    assert md5s[0] == md5s[1]
