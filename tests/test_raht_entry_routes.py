"""Every attribute-RAHT entry point of the C ABI: argument checks (CPU, before
any device is looked for) and, on the GPU, bit-exact results of the entries
the other tests do not reach -- device-pointer slices and multi-attribute
calls, point qp offsets, batches with degenerate units, and the symbol
encoder -- against the oracle or a host entry pinned to it."""
import ctypes as C

import numpy as np
import pytest

from pcc_testlib import (cloud_lidar, cloud_random, cloud_shell, make_params, make_qpset,
                         oracle_raht, sort_cloud)

INVALID = 1  # PCCB200_ERR_INVALID_ARG
FAKE = 0x1000  # never dereferenced: every call below fails its checks first
AC_QPS = [[(c % 3 - 1, (c + 1) % 3 - 1) for c in range(7)], [(1, 0)] * 7]


@pytest.fixture(scope="module")
def pb():
    import pcc_attr_b200 as pb

    pb.lib()
    return pb


def _pods(pb, params, qpset):
    return (pb.RahtParams.from_buffer_copy(bytes(params)),
            pb.QpSet.from_buffer_copy(bytes(qpset)))


def _no_gpu():
    import torch

    return not torch.cuda.is_available()


def _i32(*v):
    return (C.c_int32 * len(v))(*v)


def _ptrs(*v):
    return (C.c_void_p * len(v))(*v)


# -------------------------------------------------------------------- CPU ----

def _single_calls(pb):
    """(name, call(xyz, attrs, coeffs, A, n, bitdepth)) for the one-attribute entries"""
    lib = pb.lib()
    p, q = _pods(pb, make_params(), make_qpset())
    P, Q = C.byref(p), C.byref(q)

    def plain(fn):
        return lambda x, a, c, A, n, bd: fn(P, Q, None, x, a, C.c_int32(A), C.c_int32(n),
                                            C.c_int32(bd), c)

    def slices(fn):
        return lambda x, a, c, A, n, bd: fn(P, Q, None, x, a, C.c_int32(A), C.c_int32(bd),
                                            (C.c_int64 * 2)(0, n), C.c_int32(1), c)

    def symbols(x, a, c, A, n, bd):
        cnt, tail = C.c_int32(0), C.c_int32(0)
        return lib.pccb200_attr_raht_encode_symbols(
            P, Q, None, x, a, C.c_int32(A), C.c_int32(n), C.c_int32(bd), C.c_void_p(FAKE), c,
            C.c_void_p(FAKE), C.byref(cnt), C.byref(tail))

    return [("encode", plain(lib.pccb200_attr_raht_encode)),
            ("decode", plain(lib.pccb200_attr_raht_decode)),
            ("encode_slices", slices(lib.pccb200_attr_raht_encode_slices)),
            ("encode_slices_dev", slices(lib.pccb200_attr_raht_encode_slices_dev)),
            ("decode_slices_dev", slices(lib.pccb200_attr_raht_decode_slices_dev)),
            ("encode_symbols", symbols)]


def test_single_attribute_entries_check_arguments(pb):
    """null arrays, no points, 0 or 4 components, bit depth 0 or 17 are refused
    with PCCB200_ERR_INVALID_ARG; a well-formed call without a GPU fails loudly"""
    x = C.c_void_p(FAKE)
    for name, call in _single_calls(pb):
        assert call(None, x, x, 3, 8, 8) == INVALID, name
        assert call(x, None, x, 3, 8, 8) == INVALID, name
        assert call(x, x, None, 3, 8, 8) == INVALID, name
        assert call(x, x, x, 3, 0, 8) == INVALID, name
        assert call(x, x, x, 0, 8, 8) == INVALID, name
        assert call(x, x, x, 4, 8, 8) == INVALID, name
        assert call(x, x, x, 3, 8, 0) == INVALID, name
        assert call(x, x, x, 3, 8, 17) == INVALID, name
        if name == "encode_symbols":
            assert call(x, x, x, 2, 8, 8) == INVALID, name
        if _no_gpu():
            rc = call(x, x, x, 3, 8, 8)
            assert rc not in (0, INVALID), name


def test_slice_entries_check_offsets(pb):
    """an empty slice anywhere in the list, or no slices at all, is refused"""
    lib = pb.lib()
    p, q = _pods(pb, make_params(), make_qpset())
    x = C.c_void_p(FAKE)
    for fn in (lib.pccb200_attr_raht_encode_slices, lib.pccb200_attr_raht_encode_slices_dev,
               lib.pccb200_attr_raht_decode_slices_dev):
        def call(offs, k):
            return fn(C.byref(p), C.byref(q), x, x, x, C.c_int32(3), C.c_int32(8),
                      (C.c_int64 * len(offs))(*offs), C.c_int32(k), x)

        assert call([0, 5, 5, 9], 3) == INVALID
        assert call([0, 5, 3], 2) == INVALID
        assert call([0], 0) == INVALID
        if _no_gpu():
            assert call([0, 5, 9], 2) not in (0, INVALID)


def test_raht_transform_entries_check_arguments(pb):
    lib = pb.lib()
    p, q = _pods(pb, make_params(), make_qpset())
    x = C.c_void_p(FAKE)
    for fn in (lib.pccb200_raht_forward, lib.pccb200_raht_inverse):
        def call(keys, a, c, A, n):
            return fn(C.byref(p), C.byref(q), None, keys, a, C.c_int32(A), C.c_int32(n), c)

        assert call(None, x, x, 3, 8) == INVALID
        assert call(x, None, x, 3, 8) == INVALID
        assert call(x, x, None, 3, 8) == INVALID
        assert call(x, x, x, 3, 0) == INVALID
        assert call(x, x, x, 0, 8) == INVALID
        assert call(x, x, x, 4, 8) == INVALID
        if _no_gpu():
            assert call(x, x, x, 3, 8) not in (0, INVALID)


def _multi_calls(pb):
    lib = pb.lib()
    return [lib.pccb200_attr_raht_encode_multi, lib.pccb200_attr_raht_decode_multi,
            lib.pccb200_attr_raht_encode_multi_dev, lib.pccb200_attr_raht_decode_multi_dev]


def _batch_calls(pb):
    lib = pb.lib()
    return [lib.pccb200_attr_raht_encode_multi_batch, lib.pccb200_attr_raht_decode_multi_batch,
            lib.pccb200_attr_raht_encode_multi_batch_dev, lib.pccb200_attr_raht_decode_multi_batch_dev]


def _set_cases():
    """(sets, A, bitdepths, attrs pointer list, valid?) per attribute description"""
    f = FAKE
    return [
        (2, [3, 1], [8, 8], [f, f], True),
        (1, [3], [8], [f], True),
        (0, [3], [8], [f], False),
        (3, [1, 1, 1], [8, 8, 8], [f, f, f], False),
        (2, [3, 3], [8, 8], [f, f], False),  # more than four components
        (2, [3, 0], [8, 8], [f, f], False),
        (2, [4, 0], [8, 8], [f, f], False),
        (2, [3, 1], [8, 0], [f, f], False),
        (2, [3, 1], [17, 8], [f, f], False),
        (2, [3, 1], [8, 8], [f, None], False),
    ]


def test_multi_entries_check_arguments(pb):
    p, q = _pods(pb, make_params(), make_qpset())
    QP = C.POINTER(pb.QpSet) * 3
    qp = QP(C.pointer(q), C.pointer(q), C.pointer(q))
    x = C.c_void_p(FAKE)
    for fn in _multi_calls(pb):
        def call(k, A, bd, at, co, xyz=x, n=8, qps=qp):
            return fn(C.byref(p), C.c_int32(k), qps, xyz, at, _i32(*A), _i32(*bd), C.c_int32(n), co)

        for k, A, bd, at, ok in _set_cases():
            co = _ptrs(*[FAKE] * len(at))
            if ok:
                assert call(k, A, bd, _ptrs(*at), co, xyz=None) == INVALID
                assert call(k, A, bd, None, co) == INVALID
                assert call(k, A, bd, _ptrs(*at), None) == INVALID
                assert call(k, A, bd, _ptrs(*at), _ptrs(*[None] * len(at))) == INVALID
                assert call(k, A, bd, _ptrs(*at), co, n=0) == INVALID
                assert call(k, A, bd, _ptrs(*at), co, qps=None) == INVALID
                if _no_gpu():
                    assert call(k, A, bd, _ptrs(*at), co) not in (0, INVALID)
            else:
                assert call(k, A, bd, _ptrs(*at), co) == INVALID, (k, A, bd)


def test_batch_entries_check_arguments(pb):
    p, q = _pods(pb, make_params(), make_qpset())
    QP = C.POINTER(pb.QpSet) * 3
    qp = QP(C.pointer(q), C.pointer(q), C.pointer(q))
    for fn in _batch_calls(pb):
        def call(k, A, bd, at, ns, xyz=None, co=None, units=2):
            m = len(ns)
            xyz = xyz if xyz is not None else _ptrs(*[FAKE] * m)
            co = co if co is not None else _ptrs(*[FAKE] * (m * max(k, 1)))
            return fn(C.byref(p), C.c_int32(k), qp, C.c_int32(units), xyz, at, _i32(*A),
                      _i32(*bd), _i32(*ns), co)

        for k, A, bd, at, ok in _set_cases():
            at2 = _ptrs(*(at * 2))
            if ok:
                assert call(k, A, bd, at2, [8, 5], xyz=_ptrs(FAKE, None)) == INVALID
                assert call(k, A, bd, None, [8, 5]) == INVALID
                assert call(k, A, bd, at2, [8, 0]) == INVALID
                assert call(k, A, bd, at2, [8, 5], units=0) == INVALID
                assert call(k, A, bd, at2, [8, 5], co=_ptrs(*[FAKE] * (2 * k - 1), None)) == INVALID
                if _no_gpu():
                    assert call(k, A, bd, at2, [8, 5]) not in (0, INVALID)
            else:
                assert call(k, A, bd, at2, [8, 5]) == INVALID, (k, A, bd)


# -------------------------------------------------------------------- GPU ----

def _oracle_clip(params, qpset, xyz, attrs, qpo=None, bitdepth=8):
    """oracle RAHT of one coding unit plus clip and scatter: (rec [N,A], coef [A,N])"""
    mort, a_s, order = sort_cloud(xyz, attrs)
    orec, ocoef = oracle_raht(1, params, qpset, mort, a_s,
                              qpoffs=qpo[order] if qpo is not None else None)
    exp = np.empty_like(orec)
    exp[order] = np.clip(orec, 0, (1 << bitdepth) - 1)
    return exp, ocoef


def _cuda(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
def test_slices_dev_with_qp_offsets(pb):
    """three slices coded in place on device tensors, with point qp offsets:
    each slice's reconstruction and its columns [o, o+n) of the [A, total]
    coefficient planes equal the oracle run on that slice alone"""
    import torch

    xyz, rgb = cloud_shell(60000, bits=9, seed=17)
    total = xyz.shape[0]
    qpo = np.random.default_rng(5).integers(-6, 7, size=(total, 2)).astype(np.int32)
    offs = np.array([0, 9000, 31000, total], dtype=np.int64)
    params, qpset = make_params(), make_qpset(qp=30)
    p, q = _pods(pb, params, qpset)
    dx, dq, da = _cuda(xyz), _cuda(qpo), _cuda(rgb)
    dc = torch.empty((3, total), dtype=torch.int32, device="cuda")
    pb.attr_raht_encode_dev(p, q, dx.data_ptr(), da.data_ptr(), dc.data_ptr(), total, 3,
                            d_qpoffs=dq.data_ptr(), slice_offsets=offs)
    torch.cuda.synchronize()
    rec, coef = da.cpu().numpy(), dc.cpu().numpy()
    for s in range(3):
        a, b = offs[s], offs[s + 1]
        exp, ocoef = _oracle_clip(params, qpset, xyz[a:b], rgb[a:b], qpo[a:b])
        assert np.array_equal(coef[:, a:b], ocoef), s
        assert np.array_equal(rec[a:b], exp), s
    dd = torch.zeros_like(da)
    pb.attr_raht_decode_dev(p, q, dx.data_ptr(), dd.data_ptr(), dc.data_ptr(), total, 3,
                            d_qpoffs=dq.data_ptr(), slice_offsets=offs)
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy(), rec)


@pytest.mark.gpu
def test_host_entries_with_qp_offsets(pb):
    xyz, rgb = cloud_lidar(50000, seed=23)
    n = xyz.shape[0]
    qpo = np.random.default_rng(6).integers(-6, 7, size=(n, 2)).astype(np.int32)
    params, qpset = make_params(search_range=2500), make_qpset(qp=34)
    p, q = _pods(pb, params, qpset)
    offs = np.array([0, 20000, n], dtype=np.int64)
    rec, coef = pb.attr_raht_encode(p, q, xyz, rgb, qpoffs=qpo, slice_offsets=offs)
    for s in range(2):
        a, b = offs[s], offs[s + 1]
        exp, ocoef = _oracle_clip(params, qpset, xyz[a:b], rgb[a:b], qpo[a:b])
        assert np.array_equal(coef[:, a:b], ocoef), s
        assert np.array_equal(rec[a:b], exp), s
    exp, ocoef = _oracle_clip(params, qpset, xyz, rgb, qpo)
    assert np.array_equal(pb.attr_raht_decode(p, q, xyz, ocoef, qpoffs=qpo), exp)


def _two_attrs(n, seed):
    from pcc_attr_b200.synth import texture

    xyz, rgb = cloud_shell(n, bits=9, seed=seed)
    rgb = texture(rgb, 24, seed)
    refl = texture(((rgb[:, :1] * 2 + rgb[:, 2:3]) // 3).astype(np.int32), 12, seed + 1)
    return xyz, [rgb, refl]


def _qpsets(pb, case):
    q1 = dict(qp=34, ac_qps=AC_QPS) if case == "aclayers" else dict(qp=34)
    return [pb.QpSet.from_buffer_copy(bytes(make_qpset(**q1))),
            pb.QpSet.from_buffer_copy(bytes(make_qpset(qp=28, chroma_offset=0)))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fused", "aclayers"])
def test_multi_dev_entries(pb, case):
    """one unit, colour + reflectance, device pointers == the host multi entry"""
    import torch

    xyz, attrs = _two_attrs(50000, 9)
    n = xyz.shape[0]
    p = pb.RahtParams.from_buffer_copy(bytes(make_params(search_range=500)))
    q = _qpsets(pb, case)
    recs, coefs = pb.attr_raht_encode_multi(p, q, xyz, attrs)
    dx = _cuda(xyz)
    da = [_cuda(a) for a in attrs]
    dc = [torch.empty((a.shape[1], n), dtype=torch.int32, device="cuda") for a in attrs]
    pb.attr_raht_encode_multi_dev(p, q, dx.data_ptr(), [a.data_ptr() for a in da],
                                  [c.data_ptr() for c in dc], n, [3, 1])
    torch.cuda.synchronize()
    for s in range(2):
        assert np.array_equal(dc[s].cpu().numpy(), coefs[s]), (case, s)
        assert np.array_equal(da[s].cpu().numpy(), recs[s]), (case, s)
    dd = [torch.zeros_like(a) for a in da]
    QP = C.POINTER(pb.QpSet) * 2
    pb._check(pb.lib().pccb200_attr_raht_decode_multi_dev(
        C.byref(p), C.c_int32(2), QP(*[C.pointer(x) for x in q]), C.c_void_p(dx.data_ptr()),
        _ptrs(*[d.data_ptr() for d in dd]), _i32(3, 1), _i32(8, 8), C.c_int32(n),
        _ptrs(*[c.data_ptr() for c in dc])))
    torch.cuda.synchronize()
    for s in range(2):
        assert np.array_equal(dd[s].cpu().numpy(), recs[s]), (case, s)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fused", "aclayers"])
def test_multi_batch_dev_degenerate_units(pb, case):
    """a batch on device pointers with a 1-point, a 2-point and an all-coincident
    unit among ordinary ones == the host batch entry on the same inputs"""
    import torch

    rng = np.random.default_rng(12)
    units = []
    for xyz in (cloud_random(1, 6, seed=1)[0], cloud_random(2, 6, seed=2)[0],
                np.tile(np.array([[7, 3, 9]], dtype=np.int32), (5, 1))):
        units.append((xyz, [rng.integers(0, 256, size=(xyz.shape[0], 3)).astype(np.int32),
                            rng.integers(0, 256, size=(xyz.shape[0], 1)).astype(np.int32)]))
    units += [_two_attrs(20000, 30), _two_attrs(8000, 31)]
    p = pb.RahtParams.from_buffer_copy(bytes(make_params(search_range=500)))
    q = _qpsets(pb, case)
    recs, coefs = pb.attr_raht_encode_multi_batch(p, q, [x for x, _ in units],
                                                  [a for _, a in units])
    dx = [_cuda(x) for x, _ in units]
    da = [[_cuda(a) for a in at] for _, at in units]
    dc = [[torch.empty((a.shape[1], a.shape[0]), dtype=torch.int32, device="cuda") for a in at]
          for _, at in units]
    ns = [x.shape[0] for x, _ in units]
    pb.attr_raht_multi_batch_dev(True, p, q, [x.data_ptr() for x in dx],
                                 [[a.data_ptr() for a in u] for u in da],
                                 [[c.data_ptr() for c in u] for u in dc], ns, [3, 1])
    torch.cuda.synchronize()
    for u in range(len(units)):
        for s in range(2):
            assert np.array_equal(dc[u][s].cpu().numpy(), coefs[u][s]), (case, u, s)
            assert np.array_equal(da[u][s].cpu().numpy(), recs[u][s]), (case, u, s)
    dd = [[torch.zeros_like(a) for a in u] for u in da]
    pb.attr_raht_multi_batch_dev(False, p, q, [x.data_ptr() for x in dx],
                                 [[a.data_ptr() for a in u] for u in dd],
                                 [[c.data_ptr() for c in u] for u in dc], ns, [3, 1])
    torch.cuda.synchronize()
    dec = pb.attr_raht_decode_multi_batch(p, q, [x for x, _ in units], coefs)
    for u in range(len(units)):
        for s in range(2):
            assert np.array_equal(dd[u][s].cpu().numpy(), dec[u][s]), (case, u, s)
            assert np.array_equal(dec[u][s], recs[u][s]), (case, u, s)


@pytest.mark.gpu
def test_encode_symbols_with_qp_offsets(pb):
    xyz, rgb = cloud_shell(40000, bits=9, seed=21)
    qpo = np.random.default_rng(8).integers(-6, 7, size=(xyz.shape[0], 2)).astype(np.int32)
    p, q = _pods(pb, make_params(), make_qpset(qp=30))
    rec, coef = pb.attr_raht_encode(p, q, xyz, rgb, qpoffs=qpo)
    runs, values, ctx, tail = pb.coeff_symbols(coef)
    srec, sruns, svalues, sctx, stail = pb.attr_raht_encode_symbols(p, q, xyz, rgb, qpoffs=qpo)
    assert np.array_equal(srec, rec)
    assert np.array_equal(sruns, runs) and np.array_equal(svalues, values)
    assert np.array_equal(sctx, ctx) and stail == tail
