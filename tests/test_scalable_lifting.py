"""Scalable lifting (aps.scalable_lifting_enabled_flag): the octree levels of
detail with neighbour pruning and concatenated layers, partial decoding
(minGeomNodeSizeLog2 > 0), and the lifting coder on them.

CPU: the kernel bodies run on the host (tests/emu/emu_scalable.cpp through
exec_host.h) against the reference's own AttributeLods::generate and lifting
encoder / decoder (oracle/ref_shim_scalable_*.cpp, built by
oracle/scalable.mk), live when oracle/_ref/libtmc13_scalable.so is built, else
against the results recorded in tests/golden/scalable_golden.npz
(tests/golden/make_scalable_golden.py).  GPU: the library's entries against the
same results, bit-exact."""
import atexit
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))
sys.path.insert(0, HERE)

import pcc_attr_b200 as pb  # noqa: E402
import scalable_cases as sc  # noqa: E402
from pcc_testlib import _pp, _ptr  # noqa: E402

INVALID_ARG = 1
GOLDEN = os.path.join(HERE, "golden", "scalable_golden.npz")


def _golden():
    return np.load(GOLDEN)


def _live():
    return os.path.exists(sc.REF_LIB)


def reference_lod(name):
    """(preds, indexes, npl) of case `name`: the compiled reference, else the golden"""
    if _live():
        return sc.ref_lod(*sc.lod_case(name))
    g = _golden()
    return g[f"lod/{name}/preds"], g[f"lod/{name}/indexes"], g[f"lod/{name}/npl"]


def reference_encode(name, a):
    """(values, recon, lcp) of the reference's scalable lifting encoder, lift case `name`"""
    if _live():
        lp, rng, xyz, attrs = sc.lift_case(name, a)
        return sc.ref_encode(lp, rng, xyz, attrs)
    g = _golden()
    return tuple(g[f"enc/{name}/{a}/{k}"] for k in ("values", "recon", "lcp"))


def reference_partial_decode(name, a):
    if _live():
        return sc.ref_partial_decode(name, a)
    return _golden()[f"dec/{name}/{a}/recon"]


_emu = None


def load_emu():
    """tests/emu/emu_scalable.cpp built for the host (once per process, in a temporary directory)"""
    global _emu
    if _emu is None:
        emu_dir = os.path.join(HERE, "emu")
        tmp = tempfile.mkdtemp(prefix="emu_scalable_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libemu_scalable.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-x", "c++",
                               "-I" + os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "csrc"),
                               "-I" + os.path.join(ROOT, "include"), "-I" + emu_dir,
                               os.path.join(emu_dir, "emu_scalable.cpp"), "-o", so])
        _emu = C.CDLL(so)
    return _emu


def emu_lod(lp, scal, xyz):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    n = xyz.shape[0]
    preds = np.zeros(n, dtype=pb.PREDICTOR_DTYPE)
    indexes = np.zeros(n, dtype=np.uint32)
    npl = np.zeros(pb.MAX_LODS, dtype=np.uint32)
    cnt = C.c_int32(0)
    rc = load_emu().emu_lod_build_scalable(C.byref(lp), C.byref(scal), _ptr(xyz, C.c_int32),
                                           C.c_int(n), _pp(preds), _ptr(indexes, C.c_uint32),
                                           _ptr(npl, C.c_uint32), C.byref(cnt))
    assert rc == 0, rc
    return preds, indexes, npl[:cnt.value].copy()


def emu_lift(forward, lp, scal, qpset, lcp_enabled, xyz, data, lcp=None):
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    n = xyz.shape[0]
    data = np.ascontiguousarray(data, dtype=np.int32).reshape(n, -1)
    a = data.shape[1]
    attrs = data.copy() if forward else np.zeros_like(data)
    values = np.zeros_like(data) if forward else data.copy()
    row = np.zeros(pb.MAX_LODS, dtype=np.int8)
    if lcp is not None:
        row[:len(lcp)] = lcp
    rc = load_emu().emu_lift_scalable(C.c_int(1 if forward else 0), C.byref(lp), C.byref(scal),
                                      C.byref(qpset), C.c_int(lcp_enabled), _ptr(xyz, C.c_int32),
                                      C.c_int(n), _ptr(attrs, C.c_int32), C.c_int(a), C.c_int(8),
                                      _ptr(values, C.c_int32), _ptr(row, C.c_int8))
    assert rc == 0, rc
    return (values, attrs, row[:pb.SCALABLE_LODS].copy()) if forward else attrs


def _same(got, exp):
    for g, e in zip(got, exp):
        assert np.array_equal(g, e)


# --------------------------------------------------------------------------
# CPU

def test_cases_cover_both_concatenation_regimes():
    """Some clouds stop concatenating layers at the first level, others
    concatenate several levels (PCCTMC3Common.h:2377-2406)."""
    seen = {}
    for name in sc.LOD_CASES:
        lp, scal, xyz = sc.lod_case(name)
        npl = reference_lod(name)[2]
        seen[name] = sc.concatenated_levels(npl, xyz.shape[0], scal)
    for name in sc.STOPS_AT_FIRST:
        assert seen[name] == 0, (name, seen[name])
    for name in sc.CONCATENATES_SEVERAL:
        assert seen[name] >= 2, (name, seen[name])


@pytest.mark.parametrize("name", sc.LOD_CASES)
def test_emulated_lod_build_equals_reference(name):
    """predictors, indexes and numPointsInLod of the kernel bodies (host loops)"""
    lp, scal, xyz = sc.lod_case(name)
    _same(emu_lod(lp, scal, xyz), reference_lod(name))


@pytest.mark.parametrize("name", sc.LIFT_CASES)
@pytest.mark.parametrize("a", [3, 1])
def test_emulated_lift_encode_equals_reference(name, a):
    """values, reconstruction and LCP coefficients of the encoder; the decoder of
    the encoder's values gives its reconstruction back"""
    lp, rng, xyz, attrs = sc.lift_case(name, a)
    scal = pb.LodScalable(rng, 0, 0, 0)
    q = sc.qpset()
    got = emu_lift(True, lp, scal, q, a == 3, xyz, attrs)
    _same(got, reference_encode(name, a))
    dec = emu_lift(False, lp, scal, q, a == 3, xyz, got[0], got[2])
    assert np.array_equal(dec, got[1])


@pytest.mark.parametrize("name", sc.PARTIAL_CASES)
@pytest.mark.parametrize("a", [3, 1])
def test_emulated_partial_decode_equals_reference(name, a):
    """decoder with minGeomNodeSizeLog2 > 0 and geom_num_points > n: levels of
    detail from the partial cloud, computeQuantizationWeightsScalable with the
    decoder's arguments"""
    lp, scal, xyz, values, lcp = sc.partial_case(name, a)
    got = emu_lift(False, lp, scal, sc.qpset(), a == 3, xyz, values, lcp)
    assert np.array_equal(got, reference_partial_decode(name, a))


def _scalable_call(fn, lods, scals, n_units=1, a=3, lcp_row=True, xyz_null=False):
    k = 1
    xyz = np.zeros((4, 3), dtype=np.int32)
    buf = np.zeros((4, a), dtype=np.int32)
    vals = np.zeros((4, a), dtype=np.int32)
    row = np.zeros(pb.MAX_LODS, dtype=np.int8)
    q = sc.qpset()
    VP = C.c_void_p * (n_units * k)
    return fn(C.c_int32(n_units), (C.POINTER(pb.LodParams) * n_units)(*[C.pointer(l) for l in lods]),
              scals, C.c_int32(k), (C.POINTER(pb.QpSet) * k)(C.pointer(q)), (C.c_int32 * k)(1),
              (C.c_void_p * n_units)(*[None if xyz_null else xyz.ctypes.data] * n_units),
              (C.c_int32 * n_units)(*[4] * n_units), VP(*[buf.ctypes.data] * n_units),
              (C.c_int32 * k)(a), (C.c_int32 * k)(8), VP(*[vals.ctypes.data] * n_units),
              VP(*[row.ctypes.data if lcp_row else None] * n_units))


def test_malformed_arguments_need_no_device():
    """Every malformed argument of the scalable entries returns
    PCCB200_ERR_INVALID_ARG before a device is looked up."""
    L = pb.lib()
    good = sc.lod_params()
    bad_dec = sc.lod_params()
    bad_dec.lod_decimation_type = 1
    S = pb.LodScalable
    one = lambda s: (S * 1)(s)  # noqa: E731
    for fn in (L.pccb200_attr_lift_encode_scalable, L.pccb200_attr_lift_decode_scalable,
               L.pccb200_attr_lift_encode_scalable_dev, L.pccb200_attr_lift_decode_scalable_dev):
        assert _scalable_call(fn, [bad_dec], one(S(6, 0, 0, 0))) == INVALID_ARG
        assert _scalable_call(fn, [good], one(S(0, 0, 0, 0))) == INVALID_ARG
        assert _scalable_call(fn, [good], one(S(6, 0, 3, 0))) == INVALID_ARG  # geom_num_points < n
        assert _scalable_call(fn, [good], one(S(6, 21, 0, 0))) == INVALID_ARG
        assert _scalable_call(fn, [good], one(S(6, 0, 0, 1))) == INVALID_ARG
        assert _scalable_call(fn, [good], None) == INVALID_ARG
        assert _scalable_call(fn, [good], one(S(6, 0, 0, 0)), xyz_null=True) == INVALID_ARG
    # the encoder codes whole slices
    for fn in (L.pccb200_attr_lift_encode_scalable, L.pccb200_attr_lift_encode_scalable_dev):
        assert _scalable_call(fn, [good], one(S(6, 1, 0, 0))) == INVALID_ARG
        assert _scalable_call(fn, [good], one(S(6, 0, 9, 0))) == INVALID_ARG
    xyz = np.zeros((4, 3), dtype=np.int32)
    preds = np.zeros(4, dtype=pb.PREDICTOR_DTYPE)
    idx = np.zeros(4, dtype=np.uint32)
    npl = np.zeros(pb.MAX_LODS, dtype=np.uint32)
    cnt = C.c_int32(0)
    for lp, s in ((bad_dec, S(6, 0, 0, 0)), (good, S(0, 0, 0, 0)), (good, S(6, 0, 2, 0))):
        assert L.pccb200_lod_build_scalable(C.byref(lp), C.byref(s), _ptr(xyz, C.c_int32),
                                            C.c_int32(4), _pp(preds), _ptr(idx, C.c_uint32),
                                            _ptr(npl, C.c_uint32), C.byref(cnt)) == INVALID_ARG
    assert L.pccb200_lod_build_scalable(C.byref(good), None, _ptr(xyz, C.c_int32), C.c_int32(4),
                                        _pp(preds), _ptr(idx, C.c_uint32), _ptr(npl, C.c_uint32),
                                        C.byref(cnt)) == INVALID_ARG


def test_abi_struct_layout():
    assert C.sizeof(pb.LodScalable) == 24
    assert C.sizeof(pb.LodParams) == 4 * (2 + pb.MAX_LODS + 6 + 3 + 1)


# --------------------------------------------------------------------------
# GPU

@pytest.mark.gpu
@pytest.mark.parametrize("name", sc.LOD_CASES)
def test_gpu_lod_build_equals_reference(name):
    lp, scal, xyz = sc.lod_case(name)
    _same(pb.lod_build_scalable(lp, scal, xyz), reference_lod(name))


@pytest.mark.gpu
def test_gpu_lod_build_million_points():
    """a 1M-point LiDAR-like slice: the device build equals the kernel bodies run on the host"""
    lp = sc.lod_params()
    xyz = sc.million_point_slice()
    scal = pb.LodScalable(6, 0, 0, 0)
    _same(pb.lod_build_scalable(lp, scal, xyz), emu_lod(lp, scal, xyz))


def _units(a_sets=(3, 1)):
    """three units of the lift cases, colour + reflectance"""
    units = []
    for name in sc.LIFT_CASES:
        lp, rng, xyz, rgb = sc.lift_case(name, 3)
        _, _, _, refl = sc.lift_case(name, 1)
        units.append((name, lp, pb.LodScalable(rng, 0, 0, 0), xyz, [rgb, refl]))
    return units


@pytest.mark.gpu
def test_gpu_lift_encode_equals_reference_and_decodes():
    """several units, colour (with LCP) + reflectance in one call, host pointers;
    each set equals its one-set call; the decoder reproduces the reconstruction"""
    units = _units()
    q = [sc.qpset(), sc.qpset()]
    lods = [u[1] for u in units]
    scals = [u[2] for u in units]
    xyzs = [u[3] for u in units]
    vals, recs, lcps = pb.attr_lift_scalable(True, lods, scals, q, xyzs, [u[4] for u in units],
                                             lcp_enabled=[1, 0])
    for i, (name, *_rest) in enumerate(units):
        for s, a in enumerate((3, 1)):
            ev, er, el = reference_encode(name, a)
            assert np.array_equal(vals[i][s], ev) and np.array_equal(recs[i][s], er)
            if a == 3:
                assert np.array_equal(lcps[i][s], el)
    # one set per call
    for s in range(2):
        v1, r1, l1 = pb.attr_lift_scalable(True, lods, scals, [q[s]], xyzs,
                                           [[u[4][s]] for u in units], lcp_enabled=[1 - s])
        for i in range(len(units)):
            assert np.array_equal(v1[i][0], vals[i][s]) and np.array_equal(r1[i][0], recs[i][s])
            assert np.array_equal(l1[i][0], lcps[i][s])
    dec = pb.attr_lift_scalable(False, lods, scals, q, xyzs, vals, lcp_enabled=[1, 0],
                                lcps=[[l[0], None] for l in lcps])
    for i in range(len(units)):
        for s in range(2):
            assert np.array_equal(dec[i][s], recs[i][s])


@pytest.mark.gpu
def test_gpu_lift_device_pointers():
    """the _dev entries give the host entries' results"""
    import torch

    units = _units()
    q = [sc.qpset(), sc.qpset()]
    lods = [u[1] for u in units]
    scals = [u[2] for u in units]
    xyzs = [u[3] for u in units]
    vals, recs, lcps = pb.attr_lift_scalable(True, lods, scals, q, xyzs, [u[4] for u in units],
                                             lcp_enabled=[1, 0])
    dx = [torch.from_numpy(np.ascontiguousarray(x, dtype=np.int32)).cuda() for x in xyzs]
    da = [[torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32).reshape(len(x), -1)).cuda()
           for a in u[4]] for x, u in zip(xyzs, units)]
    dv = [[torch.zeros_like(a) for a in u] for u in da]
    rows = np.zeros((len(units), 2, pb.MAX_LODS), dtype=np.int8)
    torch.cuda.synchronize()
    pb.attr_lift_scalable_dev(True, lods, scals, q, dx, da, dv, rows, lcp_enabled=[1, 0])
    for i in range(len(units)):
        for s in range(2):
            assert np.array_equal(dv[i][s].cpu().numpy(), vals[i][s])
            assert np.array_equal(da[i][s].cpu().numpy(), recs[i][s])
        assert np.array_equal(rows[i, 0, :pb.SCALABLE_LODS], lcps[i][0])
    out = [[torch.zeros_like(a) for a in u] for u in da]
    pb.attr_lift_scalable_dev(False, lods, scals, q, dx, out, dv, rows, lcp_enabled=[1, 0])
    for i in range(len(units)):
        for s in range(2):
            assert np.array_equal(out[i][s].cpu().numpy(), recs[i][s])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sc.PARTIAL_CASES)
def test_gpu_partial_decode_equals_reference(name):
    for a in (3, 1):
        lp, scal, xyz, values, lcp = sc.partial_case(name, a)
        got = pb.attr_lift_scalable(False, [lp], [scal], [sc.qpset()], [xyz], [[values]],
                                    lcp_enabled=[int(a == 3)], lcps=[[lcp]])
        assert np.array_equal(got[0][0], reference_partial_decode(name, a))


@pytest.mark.gpu
def test_whole_codec_scalable_lifting(tmp_path):
    """tmc3 with the drop-in LoD build against the unmodified tmc3, scalable
    lifting: bitstream, encoder reconstruction and decoder output md5-identical;
    then a partial decode (--decodeMaxPoints below the point count, so that
    minGeomNodeSizeLog2 > 0) of the reference's bitstream by both."""
    import codec_harness as ch

    if not (os.path.exists(ch.REF_BIN) and os.path.exists(ch.B200_BIN)):
        pytest.skip("oracle/_ref/tmc3_{ref,b200} not built (make -C oracle codec)")
    from pcc_attr_b200.synth import cloud_shell

    xyz, rgb = cloud_shell(60000, bits=10, seed=12)
    ply = str(tmp_path / "in.ply")
    ch.write_ply(ply, xyz, rgb)

    def md5(p):
        return hashlib.md5(open(p, "rb").read()).hexdigest()

    flags = ch.lod_flags(qp=34, transform_type=2) + [
        "--aps_scalable_enable_flag=1", "--positionQpMultiplierLog2=3", "--pointCountMetadata=1"]
    out = {}
    for name, binary in (("ref", ch.REF_BIN), ("b200", ch.B200_BIN)):
        b, r = str(tmp_path / f"{name}.bin"), str(tmp_path / f"{name}_rec.ply")
        rc, log = ch.encode(binary, ply, b, r, flags=flags)
        assert rc == 0, log[-2000:]
        out[name] = (b, r)
    assert md5(out["ref"][0]) == md5(out["b200"][0]), "bitstreams differ"
    assert md5(out["ref"][1]) == md5(out["b200"][1]), "encoder reconstructions differ"
    d_ref, d_b200 = str(tmp_path / "dref.ply"), str(tmp_path / "db200.ply")
    assert ch.decode(ch.REF_BIN, out["ref"][0], d_ref)[0] == 0
    rc, log = ch.decode(ch.B200_BIN, out["ref"][0], d_b200)
    assert rc == 0, log[-2000:]
    assert md5(d_ref) == md5(d_b200) == md5(out["ref"][1])

    def partial(binary, path):
        cmd = [binary, "--mode=1", f"--compressedStreamPath={out['ref'][0]}",
               f"--reconstructedDataPath={path}", "--convertPlyColourspace=1",
               f"--decodeMaxPoints={xyz.shape[0] // 4}"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        return r.returncode, r.stdout

    p_ref, p_b200 = str(tmp_path / "pref.ply"), str(tmp_path / "pb200.ply")
    rc, log = partial(ch.REF_BIN, p_ref)
    if rc != 0:
        pytest.skip("the reference decoder rejects --decodeMaxPoints on this stream: " + log[-300:])
    rc, log = partial(ch.B200_BIN, p_b200)
    assert rc == 0, log[-2000:]
    assert md5(p_ref) == md5(p_b200)
