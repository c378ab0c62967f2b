"""Every attribute-lifting entry point of the C ABI: argument checks (CPU,
before any device is looked for) and, on the GPU, bit-exact results of the
routes the other tests do not reach -- host-pointer slices, point qp offsets
(single, device-pointer slices and handle entries) and one-component handle
calls with LCP enabled -- against the oracle chain."""
import ctypes as C

import numpy as np
import pytest

from pcc_testlib import (MAX_LODS, cloud_random, cloud_shell, finish_lift_recon, make_lod_params,
                         make_qpset, oracle_lcp_coeffs, oracle_lift, oracle_lift_encode,
                         oracle_lift_quant, oracle_lod_build, oracle_quant_weights)

INVALID = 1  # PCCB200_ERR_INVALID_ARG
FAKE = 0x1000  # never dereferenced: no call below reaches a device


@pytest.fixture(scope="module")
def pb():
    import pcc_attr_b200 as pb

    pb.lib()
    return pb


def _no_gpu():
    import torch

    return not torch.cuda.is_available()


def _pods(pb, lod_params, qpset):
    return (pb.LodParams.from_buffer_copy(bytes(lod_params)),
            pb.QpSet.from_buffer_copy(bytes(qpset)))


def _p(a, t=C.c_int32):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


# -------------------------------------------------------------------- CPU ----

def _calls(pb, handle=None):
    """(name, forward, kind, call) for the eight pccb200_attr_lift_* entries.
    call(**kw) makes a well-formed call with one argument replaced: lod,
    handle, qpset, xyz, attrs, values, lcp (pointers), A, n, bd, offs."""
    lib = pb.lib()
    lp, q = _pods(pb, make_lod_params(levels=4), make_qpset())
    x = C.c_void_p(FAKE)
    lcp = (C.c_int8 * (4 * MAX_LODS))()  # (the decoders read it on the calling thread)

    def args(kw):
        a = dict(lod=C.byref(lp), handle=handle, qpset=C.byref(q), xyz=x, attrs=x, values=x,
                 lcp=lcp, A=3, n=8, bd=8, offs=None)
        a.update(kw)
        if a["offs"] is None:
            a["offs"] = [0, a["n"]]
        return a

    def single(fn):
        def call(**kw):
            a = args(kw)
            return fn(a["lod"], a["qpset"], C.c_int32(1), None, a["xyz"], a["attrs"],
                      C.c_int32(a["A"]), C.c_int32(a["n"]), C.c_int32(a["bd"]), a["values"],
                      a["lcp"])
        return call

    def slices(fn):
        def call(**kw):
            a = args(kw)
            o = a["offs"]
            return fn(a["lod"], a["qpset"], C.c_int32(1), None, a["xyz"], a["attrs"],
                      C.c_int32(a["A"]), C.c_int32(a["bd"]), (C.c_int64 * len(o))(*o),
                      C.c_int32(len(o) - 1), a["values"], a["lcp"])
        return call

    def lod(fn):
        def call(**kw):
            a = args(kw)
            return fn(a["handle"], a["qpset"], C.c_int32(1), None, a["attrs"], C.c_int32(a["A"]),
                      C.c_int32(a["bd"]), a["values"], a["lcp"])
        return call

    return [("encode", True, "single", single(lib.pccb200_attr_lift_encode)),
            ("decode", False, "single", single(lib.pccb200_attr_lift_decode)),
            ("encode_slices", True, "slices", slices(lib.pccb200_attr_lift_encode_slices)),
            ("decode_slices", False, "slices", slices(lib.pccb200_attr_lift_decode_slices)),
            ("encode_slices_dev", True, "slices", slices(lib.pccb200_attr_lift_encode_slices_dev)),
            ("decode_slices_dev", False, "slices", slices(lib.pccb200_attr_lift_decode_slices_dev)),
            ("encode_lod", True, "lod", lod(lib.pccb200_attr_lift_encode_lod)),
            ("decode_lod", False, "lod", lod(lib.pccb200_attr_lift_decode_lod))]


def _assert_refused(name, forward, kind, call):
    """null arrays, 0 / 2 / 4 components, bit depth 0 or 17 and, decoding with
    LCP enabled and three components, a null lcp are refused"""
    bad = [dict(qpset=None), dict(attrs=None), dict(values=None), dict(A=0), dict(A=2),
           dict(A=4), dict(bd=0), dict(bd=17)]
    if kind != "lod":
        bad += [dict(lod=None), dict(xyz=None), dict(n=0)]
    if kind == "slices":  # an empty slice, offsets that go backwards, no slices
        bad += [dict(offs=[0, 5, 5, 9]), dict(offs=[0, 5, 3]), dict(offs=[0])]
    if not forward:
        bad.append(dict(lcp=None))
    for kw in bad:
        assert call(**kw) == INVALID, (name, kw)


def test_lift_entries_check_arguments(pb):
    """each refusal returns PCCB200_ERR_INVALID_ARG; a well-formed call
    without a GPU fails loudly"""
    for name, forward, kind, call in _calls(pb):
        if kind == "lod":  # (a handle needs a device: null here)
            assert call() == INVALID, name
            continue
        _assert_refused(name, forward, kind, call)
        if _no_gpu():
            assert call() not in (0, INVALID), name
            if kind == "slices":
                assert call(offs=[0, 5, 9]) not in (0, INVALID), name


def test_lod_handle_queries_refuse_null(pb):
    lib = pb.lib()
    lp, _ = _pods(pb, make_lod_params(), make_qpset())
    n, cnt = C.c_int32(0), C.c_int32(0)
    assert lib.pccb200_lod_info(None, C.byref(n), C.byref(cnt), None) == INVALID
    assert lib.pccb200_lod_reusable(None, C.byref(lp)) == 0


# -------------------------------------------------------------------- GPU ----

class _Handle:
    def __init__(self, pb, lp, xyz):
        self.lib = pb.lib()
        self.h = C.c_void_p()
        self.xyz = np.ascontiguousarray(xyz, dtype=np.int32)
        pb._check(self.lib.pccb200_lod_create(C.byref(lp), _p(self.xyz), C.c_int32(len(xyz)),
                                              C.byref(self.h)))

    def __enter__(self):
        return self.h

    def __exit__(self, *exc):
        self.lib.pccb200_lod_destroy(self.h)


@pytest.mark.gpu
def test_handle_entries_check_arguments(pb):
    xyz, _ = cloud_random(500, 8, seed=3)
    lp, _ = _pods(pb, make_lod_params(levels=4), make_qpset())
    with _Handle(pb, lp, xyz) as h:
        for name, forward, kind, call in _calls(pb, handle=h):
            if kind == "lod":
                _assert_refused(name, forward, kind, call)


def _oracle_lift_qpo(lod_params, qpset, xyz, attrs, qpo):
    """oracle_lift_encode with LCP enabled and point qp offsets ([N,2], point
    order; the quantiser reads them in predictor order)"""
    preds, indexes, npl = oracle_lod_build(lod_params, xyz)
    qw = oracle_quant_weights(preds)
    fwd = oracle_lift(1, preds, qw, npl, attrs[indexes].astype(np.int64) << 8)
    lcp = np.zeros(lod_params.num_detail_levels, dtype=np.int8)
    if attrs.shape[1] == 3:
        lcp = oracle_lcp_coeffs(fwd, npl, lod_params.num_detail_levels)
    rec_coef, values = oracle_lift_quant(1, qpset, qw, npl, fwd, lcp=lcp,
                                         qpo=np.ascontiguousarray(qpo[indexes], dtype=np.int32))
    out = np.zeros_like(attrs)
    out[indexes] = finish_lift_recon(oracle_lift(0, preds, qw, npl, rec_coef), 8)
    return values, out, lcp


def _cuda(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
def test_host_slices_against_oracle(pb):
    """three slices, one of 48 points, through the host-pointer slices entry:
    each slice's values, reconstruction and LCP row equal the oracle run on
    that slice alone; the decoder entry inverts it"""
    xyz, rgb = cloud_shell(50000, bits=9, seed=41)
    total = xyz.shape[0]
    offs = np.array([0, 30000, 30048, total], dtype=np.int64)
    tl = make_lod_params(levels=6), make_qpset(qp=30, fixed_point_qp_offset=24)
    lp, q = _pods(pb, *tl)
    lib = pb.lib()
    rec = rgb.copy()
    vals = np.zeros_like(rgb)
    lcp = np.zeros((3, MAX_LODS), dtype=np.int8)
    pb._check(lib.pccb200_attr_lift_encode_slices(
        C.byref(lp), C.byref(q), C.c_int32(1), None, _p(xyz), _p(rec), C.c_int32(3), C.c_int32(8),
        _p(offs, C.c_int64), C.c_int32(3), _p(vals), _p(lcp, C.c_int8)))
    for s in range(3):
        a, b = offs[s], offs[s + 1]
        ov, orec, ol = oracle_lift_encode(*tl, 1, xyz[a:b], rgb[a:b])
        assert np.array_equal(vals[a:b], ov), s
        assert np.array_equal(rec[a:b], orec), s
        assert np.array_equal(lcp[s, :6], ol) and not lcp[s, 6:].any(), s
    dec = np.zeros_like(rgb)
    pb._check(lib.pccb200_attr_lift_decode_slices(
        C.byref(lp), C.byref(q), C.c_int32(1), None, _p(xyz), _p(dec), C.c_int32(3), C.c_int32(8),
        _p(offs, C.c_int64), C.c_int32(3), _p(vals), _p(lcp, C.c_int8)))
    assert np.array_equal(dec, rec)


@pytest.mark.gpu
def test_point_qp_offsets(pb):
    """point qp offsets through the single entries and the device-pointer
    slices entries against the oracle chain"""
    import torch

    xyz, rgb = cloud_shell(40000, bits=9, seed=43)
    n = xyz.shape[0]
    qpo = np.random.default_rng(7).integers(-6, 7, size=(n, 2)).astype(np.int32)
    tl = make_lod_params(levels=6), make_qpset(qp=30, fixed_point_qp_offset=24)
    lp, q = _pods(pb, *tl)
    ov, orec, ol = _oracle_lift_qpo(*tl, xyz, rgb, qpo)
    assert not np.array_equal(oracle_lift_encode(*tl, 1, xyz, rgb)[0], ov)  # the offsets matter
    gv, grec, gl = pb.attr_lift_encode(lp, q, xyz, rgb, lcp_enabled=1, qpoffs=qpo)
    assert np.array_equal(gv, ov) and np.array_equal(grec, orec) and np.array_equal(gl, ol)
    assert np.array_equal(pb.attr_lift_decode(lp, q, xyz, ov, lcp=ol, qpoffs=qpo), orec)

    offs = np.array([0, 15000, n], dtype=np.int64)
    dx, dq, da = _cuda(xyz), _cuda(qpo), _cuda(rgb)
    dv = torch.zeros_like(da)
    lcp = np.zeros((2, MAX_LODS), dtype=np.int8)
    pb.attr_lift_slices_dev(True, lp, q, 1, dx.data_ptr(), da.data_ptr(), 3, offs, dv.data_ptr(),
                            lcp, d_qpoffs=dq.data_ptr())
    torch.cuda.synchronize()
    rec, vals = da.cpu().numpy(), dv.cpu().numpy()
    for s in range(2):
        a, b = offs[s], offs[s + 1]
        sv, srec, sl = _oracle_lift_qpo(*tl, xyz[a:b], rgb[a:b], qpo[a:b])
        assert np.array_equal(vals[a:b], sv) and np.array_equal(rec[a:b], srec), s
        assert np.array_equal(lcp[s, :6], sl), s
    dd = torch.zeros_like(da)
    pb.attr_lift_slices_dev(False, lp, q, 1, dx.data_ptr(), dd.data_ptr(), 3, offs, dv.data_ptr(),
                            lcp, d_qpoffs=dq.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy(), rec)


@pytest.mark.gpu
def test_handle_entries_with_qp_offsets(pb):
    """the handle entries with point qp offsets and LCP enabled, colour and
    reflectance, against the oracle chain.  With one component the LCP
    coefficients are not used: the encoder writes zeros and the decoder
    accepts a null pointer."""
    xyz, rgb = cloud_shell(40000, bits=9, seed=45)
    n = xyz.shape[0]
    refl = ((rgb[:, :1] + rgb[:, 1:2]) // 2).astype(np.int32)
    qpo = np.random.default_rng(9).integers(-6, 7, size=(n, 2)).astype(np.int32)
    tl = make_lod_params(levels=6), make_qpset(qp=30, fixed_point_qp_offset=24)
    lp, q = _pods(pb, *tl)
    lib = pb.lib()
    with _Handle(pb, lp, xyz) as h:
        for attrs in (rgb, refl):
            A = attrs.shape[1]
            ov, orec, ol = _oracle_lift_qpo(*tl, xyz, attrs, qpo)
            rec = attrs.copy()
            vals = np.zeros_like(attrs)
            lcp = np.full(MAX_LODS, 99, dtype=np.int8)
            pb._check(lib.pccb200_attr_lift_encode_lod(
                h, C.byref(q), C.c_int32(1), _p(qpo), _p(rec), C.c_int32(A), C.c_int32(8),
                _p(vals), _p(lcp, C.c_int8)))
            assert np.array_equal(vals, ov) and np.array_equal(rec, orec), A
            assert np.array_equal(lcp[:6], ol) and np.all(lcp[6:] == 99), A
            dec = np.zeros_like(attrs)
            pb._check(lib.pccb200_attr_lift_decode_lod(
                h, C.byref(q), C.c_int32(1), _p(qpo), _p(dec), C.c_int32(A), C.c_int32(8),
                _p(vals), _p(lcp, C.c_int8) if A == 3 else None))
            assert np.array_equal(dec, orec), A
