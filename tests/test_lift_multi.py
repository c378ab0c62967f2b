"""Lifting several attribute sets of a slice in one pass, and many slices or
frames per call (pccb200_attr_lift_{en,de}code_multi, _multi_dev,
_multi_batch, _multi_batch_dev).  Every set's values, reconstruction and LCP
row must be bit-identical to the oracle chain run on that set alone: on the
host through the product's kernel bodies (tests/emu), and -- on a GPU --
through the C ABI."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from pcc_testlib import (MAX_LODS, ROOT, _ptr, cloud_random, cloud_shell, make_lod_params, make_qpset,
                         oracle_lift_encode)
from pcc_attr_b200.synth import texture

INVALID = 1  # PCCB200_ERR_INVALID_ARG
UNSUPPORTED = 5  # PCCB200_ERR_UNSUPPORTED

# name: (cloud, make_lod_params arguments)
CONFIGS = {
    "distance_12": ("shell", dict(levels=12)),
    "periodic_12": ("shell", dict(levels=12, decimation=1)),
    "centroid_12": ("random", dict(levels=12, decimation=2)),
    "distance_6_nodistribution": ("random", dict(levels=6, distribution=0)),
    "periodic_6": ("random", dict(levels=6, decimation=1, period=3)),
    "one_level": ("shell", dict(levels=1)),
}


def colour_qpset():
    return make_qpset(qp=30, chroma_offset=-2, fixed_point_qp_offset=24)


def refl_qpset(bits):
    return make_qpset(qp=40, chroma_offset=0, bitdepth=bits, fixed_point_qp_offset=24)


def reflectance(rgb, bits, seed):
    """a one-component attribute at `bits` bits; at 16 bits the values span 0..65535"""
    r = (rgb[:, :1].astype(np.int64) * 2 + rgb[:, 1:2]) // 3
    if bits == 16:
        rng = np.random.default_rng(seed)
        r = np.clip(r * 257 + rng.integers(-4000, 4001, size=r.shape), 0, 65535)
        r[: r.shape[0] // 50] = 65535
        r[r.shape[0] // 50: r.shape[0] // 25] = 0
        rng.shuffle(r)
    return np.ascontiguousarray(r.astype(np.int32))


def make_cloud(kind, n=20000, seed=11):
    if kind == "shell":
        xyz, rgb = cloud_shell(n, bits=9, seed=seed)
    else:
        xyz, rgb = cloud_random(n, 8, seed)
    return np.ascontiguousarray(xyz), np.ascontiguousarray(texture(rgb, 20, seed + 1).astype(np.int32))


class Set:
    """one attribute set: attributes, QpSet, lcp_enabled, bit depth"""

    def __init__(self, attrs, qpset, lcp, bits):
        self.attrs, self.qpset, self.lcp, self.bits = np.ascontiguousarray(attrs), qpset, lcp, bits


def colour_and_refl(rgb, refl_bits, seed=5):
    return [Set(rgb, colour_qpset(), 1, 8), Set(reflectance(rgb, refl_bits, seed), refl_qpset(refl_bits), 1, refl_bits)]


def oracle_per_set(lp, xyz, sets):
    """-> [(values, reconstruction, lcp)] of the oracle chain run once per set"""
    return [oracle_lift_encode(lp, s.qpset, s.lcp, xyz, s.attrs, bitdepth=s.bits) for s in sets]


_emu = None


def load_emu_multi():
    """tests/emu/emu_lift_multi.cpp built for the host (once per process, in a
    temporary directory)"""
    global _emu
    if _emu is None:
        emu_dir = os.path.join(ROOT, "tests", "emu")
        tmp = tempfile.mkdtemp(prefix="emu_lift_multi_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libemu_lift_multi.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-x", "c++",
                               "-I" + os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "csrc"),
                               "-I" + os.path.join(ROOT, "include"), "-I" + emu_dir,
                               os.path.join(emu_dir, "emu_lift_multi.cpp"), "-o", so])
        _emu = C.CDLL(so)
    return _emu


def emu_lift_multi(forward, lp, xyz, sets, values=None, lcps=None):
    """the several-set pipeline on the host.  forward: -> ([values], [recon],
    [lcp]); otherwise values[s], lcps[s] in -> ([recon]) (rc on failure)"""
    lib = load_emu_multi()
    k, n = len(sets), xyz.shape[0]
    levels = lp.num_detail_levels
    attrs = [s.attrs.copy() if forward else np.zeros_like(s.attrs) for s in sets]
    vals = [np.zeros_like(s.attrs) for s in sets] if forward else [np.ascontiguousarray(v) for v in values]
    rows = [np.zeros(MAX_LODS, dtype=np.int8) for _ in sets]
    if not forward:
        for r, l in zip(rows, lcps):
            r[:len(l)] = l
    IP = C.POINTER(C.c_int32) * k
    rc = lib.emu_lift_multi(C.c_int(1 if forward else 0), C.byref(lp), C.c_int(k),
                            (C.c_void_p * k)(*[C.addressof(s.qpset) for s in sets]),
                            (C.c_int32 * k)(*[s.lcp for s in sets]), _ptr(xyz, C.c_int32), C.c_int(n),
                            IP(*[_ptr(a, C.c_int32) for a in attrs]), (C.c_int32 * k)(*[s.attrs.shape[1] for s in sets]),
                            (C.c_int32 * k)(*[s.bits for s in sets]), IP(*[_ptr(v, C.c_int32) for v in vals]),
                            (C.POINTER(C.c_int8) * k)(*[_ptr(r, C.c_int8) for r in rows]))
    if rc:
        return rc
    if not forward:
        return attrs
    return vals, attrs, [r[:levels].copy() for r in rows]


def assert_results_equal(got, exp, what):
    """got / exp: [(values, reconstruction, lcp)] per set"""
    assert len(got) == len(exp), what
    for s, (g, e) in enumerate(zip(got, exp)):
        for name, x, y in zip(("values", "reconstruction", "lcp"), g, e):
            assert x.shape == y.shape and np.array_equal(x, y), (what, s, name, int((x != y).sum()))


def _emu_vs_oracle(lp, xyz, sets, what):
    vals, recs, lcps = emu_lift_multi(True, lp, xyz, sets)
    assert_results_equal(list(zip(vals, recs, lcps)), oracle_per_set(lp, xyz, sets), what)
    dec = emu_lift_multi(False, lp, xyz, sets, values=vals, lcps=lcps)
    for s, (d, r) in enumerate(zip(dec, recs)):
        assert np.array_equal(d, r), (what, "decode", s)


# ---- host: the several-set pipeline against the oracle --------------------------

@pytest.mark.parametrize("refl_bits", [8, 16])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_emu_multi_vs_oracle(name, refl_bits):
    kind, kw = CONFIGS[name]
    xyz, rgb = make_cloud(kind)
    lp = make_lod_params(**kw)
    _emu_vs_oracle(lp, xyz, colour_and_refl(rgb, refl_bits), name)


def test_emu_reflectance_first():
    xyz, rgb = make_cloud("shell", seed=13)
    lp = make_lod_params(levels=6)
    _emu_vs_oracle(lp, xyz, colour_and_refl(rgb, 16)[::-1], "reflectance first")


@pytest.mark.parametrize("num_sets", [3, 4])
def test_emu_three_and_four_sets(num_sets):
    """two colour sets, LCP on and off, with reflectance at 16 and 8 bits"""
    xyz, rgb = make_cloud("random", seed=17)
    rgb2 = np.ascontiguousarray(rgb[::-1])
    sets = [Set(rgb, colour_qpset(), 1, 8), Set(reflectance(rgb, 16, 3), refl_qpset(16), 0, 16),
            Set(rgb2, make_qpset(qp=34, chroma_offset=3, fixed_point_qp_offset=24), 0, 8),
            Set(reflectance(rgb, 8, 4), refl_qpset(8), 1, 8)][:num_sets]
    _emu_vs_oracle(make_lod_params(levels=12), xyz, sets, num_sets)


def test_emu_own_level_predictors_unsupported():
    """predictors that reference their own level of detail: the one-set and the
    several-set forms both refuse"""
    from pcc_testlib import emu_attr_lift, load_emu

    xyz, rgb = make_cloud("shell", n=3000)
    lp = make_lod_params(decimation=0, skip_layers=0, intra_range=128, inter_range=128)
    sets = colour_and_refl(rgb, 8)
    assert emu_lift_multi(True, lp, xyz, sets) == UNSUPPORTED
    lib = load_emu()
    lib.emu_attr_lift.restype = C.c_int
    with pytest.raises(AssertionError, match=str(UNSUPPORTED)):
        emu_attr_lift(1, lp, sets[0].qpset, 1, xyz, sets[0].attrs)


# ---- the C entries refuse malformed arguments before they look for a device ------

class _Call:
    """one well-formed call of each new entry: two units of 16 and 12 points,
    colour (LCP on) + reflectance.  Host arrays everywhere; without a device the
    *_dev entries never dereference theirs."""

    def __init__(self):
        import pcc_attr_b200 as pb

        self.pb = pb
        self.lib = pb.lib()
        self.lods = [pb.LodParams.from_buffer_copy(bytes(make_lod_params(levels=4))) for _ in range(2)]
        self.qs = [pb.QpSet.from_buffer_copy(bytes(q)) for q in (colour_qpset(), refl_qpset(8))]
        self.xyz = [np.zeros((16, 3), dtype=np.int32), np.zeros((12, 3), dtype=np.int32)]
        self.attrs = [[np.zeros((m, 3), dtype=np.int32), np.zeros((m, 1), dtype=np.int32)] for m in (16, 12)]
        self.vals = [[np.zeros_like(a) for a in u] for u in self.attrs]
        self.lcp = [[np.zeros(MAX_LODS, dtype=np.int8) for _ in u] for u in self.attrs]

    def args(self, **kw):
        a = dict(num_units=2, lods=[C.addressof(x) for x in self.lods], num_sets=2,
                 qpsets=[C.addressof(q) for q in self.qs], lcp_enabled=[1, 1],
                 xyz=[x.ctypes.data for x in self.xyz], n=[16, 12],
                 attrs=[a.ctypes.data for u in self.attrs for a in u], na=[3, 1], bd=[8, 8],
                 values=[v.ctypes.data for u in self.vals for v in u],
                 lcp=[r.ctypes.data for u in self.lcp for r in u])
        a.update(kw)
        return a

    @staticmethod
    def _arr(t, v):
        return None if v is None else (t * len(v))(*v)

    def batch(self, forward, dev=False, **kw):
        a = self.args(**kw)
        name = "encode" if forward else "decode"
        fn = getattr(self.lib, f"pccb200_attr_lift_{name}_multi_batch" + ("_dev" if dev else ""))
        A, VP, I = self._arr, C.c_void_p, C.c_int32
        return fn(I(a["num_units"]), A(VP, a["lods"]), I(a["num_sets"]), A(VP, a["qpsets"]),
                  A(I, a["lcp_enabled"]), A(VP, a["xyz"]), A(I, a["n"]), A(VP, a["attrs"]), A(I, a["na"]),
                  A(I, a["bd"]), A(VP, a["values"]), A(VP, a["lcp"]))

    def single(self, forward, dev=False, **kw):
        """unit 0 of args() through pccb200_attr_lift_*_multi(_dev)"""
        a = self.args(**kw)
        k = a["num_sets"]
        name = "encode" if forward else "decode"
        fn = getattr(self.lib, f"pccb200_attr_lift_{name}_multi" + ("_dev" if dev else ""))
        A, VP, I = self._arr, C.c_void_p, C.c_int32
        first = lambda v: None if v is None else v[:k]
        return fn(VP(a["lods"][0]) if a["lods"] else None, I(k), A(VP, a["qpsets"]), A(I, a["lcp_enabled"]),
                  VP(a["xyz"][0]) if a["xyz"] else None, I(a["n"][0]), A(VP, first(a["attrs"])), A(I, a["na"]),
                  A(I, a["bd"]), A(VP, first(a["values"])), A(VP, first(a["lcp"])))


def _malformed(c, forward):
    """(what, overrides) for every kind of malformed input"""
    a = c.args()
    bad = [
        ("null lods", dict(lods=None)),
        ("null lod of a unit", dict(lods=[a["lods"][0], None])),
        ("null qpset array", dict(qpsets=None)),
        ("null qpset of a set", dict(qpsets=[a["qpsets"][0], None])),
        ("null lcp_enabled", dict(lcp_enabled=None)),
        ("null positions", dict(xyz=None)),
        ("null positions of a unit", dict(xyz=[a["xyz"][0], None])),
        ("null point counts", dict(n=None)),
        ("null attribute array", dict(attrs=None)),
        ("null attributes of a set", dict(attrs=[a["attrs"][0], None] + a["attrs"][2:])),
        ("null component counts", dict(na=None)),
        ("null bit depths", dict(bd=None)),
        ("null value array", dict(values=None)),
        ("null values of a set", dict(values=a["values"][:1] + [None] + a["values"][2:])),
        ("null values of a set of a unit", dict(values=a["values"][:3] + [None])),
        ("num_sets 0", dict(num_sets=0)),
        ("num_sets 5", dict(num_sets=5, qpsets=a["qpsets"] * 3, lcp_enabled=[0] * 5, na=[3, 1, 1, 1, 1],
                            bd=[8] * 5, attrs=a["attrs"] * 3, values=a["values"] * 3, lcp=a["lcp"] * 3)),
        ("two components", dict(na=[3, 2])),
        ("four components", dict(na=[4, 1])),
        ("no components", dict(na=[0, 1])),
        ("bit depth 0", dict(bd=[0, 8])),
        ("bit depth 17", dict(bd=[8, 17])),
        ("no points", dict(n=[16, 0])),
        ("negative point count", dict(n=[-3, 12])),
    ]
    if not forward:
        bad += [("null lcp array with LCP", dict(lcp=None)),
                ("null lcp row of an LCP colour set", dict(lcp=[a["lcp"][0], a["lcp"][1], None, a["lcp"][3]]))]
    return bad


@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("forward", [True, False])
def test_batch_entry_argument_checks(forward, dev):
    import torch

    c = _Call()
    for what, kw in _malformed(c, forward) + [("no units", dict(num_units=0))]:
        assert c.batch(forward, dev, **kw) == INVALID, what
    # the lcp rows are optional where no set needs them
    if not torch.cuda.is_available():
        for kw in ({}, dict(lcp=None, lcp_enabled=[0, 0]), dict(lcp=[None] * 4, na=[1, 1], bd=[8, 16])):
            rc = c.batch(forward, dev, **kw)
            assert rc not in (0, INVALID), kw
            assert b"CUDA" in c.lib.pccb200_last_error() or b"device" in c.lib.pccb200_last_error()


@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("forward", [True, False])
def test_single_entry_argument_checks(forward, dev):
    """pccb200_attr_lift_*_multi(_dev): unit 0 of the same cases (a case that
    only breaks unit 1 is well-formed here)"""
    import torch

    c = _Call()
    for what, kw in _malformed(c, forward):
        if "of a unit" in what or what == "null point counts" or what == "null lods":
            continue
        kw = {"no points": dict(n=[0]), "null lcp row of an LCP colour set": dict(lcp=[None, c.args()["lcp"][1]])}.get(what, kw)
        assert c.single(forward, dev, **kw) == INVALID, what
    assert c.single(forward, dev, lods=None) == INVALID
    if not torch.cuda.is_available():
        rc = c.single(forward, dev)
        assert rc not in (0, INVALID)
        assert b"CUDA" in c.lib.pccb200_last_error() or b"device" in c.lib.pccb200_last_error()


def test_batch_refusal_names_the_unit():
    import pcc_attr_b200 as pb

    c = _Call()
    assert c.batch(True, n=[16, 0]) == INVALID
    assert b"unit 1" in pb.lib().pccb200_last_error()


def test_binding_batch_decode_without_lcp_rows_is_refused():
    """attr_lift_multi_batch decoding a colour set with LCP enabled but no LCP
    row passes a null row, which the library refuses before any device lookup"""
    import pcc_attr_b200 as pb

    c = _Call()
    vals = [[np.zeros_like(a) for a in u] for u in c.attrs]
    for lcps in (None, [[None, None], [np.zeros(4, dtype=np.int8), None]]):
        with pytest.raises(pb.PccB200Error, match="lcp coefficients missing"):
            pb.attr_lift_multi_batch(False, c.lods, c.qs, c.xyz, vals, [1, 1], [8, 8], lcps)


# ---- GPU: the C entries against the oracle and against one-set calls ---------------

def _pods(lp, sets):
    import pcc_attr_b200 as pb

    return (pb.LodParams.from_buffer_copy(bytes(lp)),
            [pb.QpSet.from_buffer_copy(bytes(s.qpset)) for s in sets])


def _gpu_multi(lp, xyz, sets):
    """-> [(values, reconstruction, lcp)] of pccb200_attr_lift_encode_multi, and
    the decoder's reconstruction"""
    import pcc_attr_b200 as pb

    glp, qs = _pods(lp, sets)
    en, bd = [s.lcp for s in sets], [s.bits for s in sets]
    vals, recs, lcps = pb.attr_lift_multi_encode(glp, qs, xyz, [s.attrs for s in sets], en, bd)
    dec = pb.attr_lift_multi_decode(glp, qs, xyz, vals, lcps, en, bd)
    return list(zip(vals, recs, lcps)), dec


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["distance_12", "centroid_12", "distance_6_nodistribution", "one_level"])
def test_gpu_multi_vs_oracle(name):
    kind, kw = CONFIGS[name]
    xyz, rgb = cloud_shell(50000, bits=9, seed=31)
    rgb = np.ascontiguousarray(texture(rgb, 20, 32).astype(np.int32))
    lp = make_lod_params(**kw)
    sets = colour_and_refl(rgb, 16)
    got, dec = _gpu_multi(lp, xyz, sets)
    assert_results_equal(got, oracle_per_set(lp, xyz, sets), name)
    for s in range(len(sets)):
        assert np.array_equal(dec[s], got[s][1]), (name, "decode", s)


@pytest.mark.gpu
def test_gpu_multi_full_size():
    """1M points of the bench frame: {RGB with LCP, reflectance} in one call is
    bit-identical to two pccb200_attr_lift_encode calls"""
    import bench
    import pcc_attr_b200 as pb

    xyz, rgb, refl = bench.make_frame(2)
    lp = make_lod_params(levels=12)
    sets = [Set(rgb, colour_qpset(), 1, 8), Set(refl, refl_qpset(8), 0, 8)]
    got, dec = _gpu_multi(lp, xyz, sets)
    glp, qs = _pods(lp, sets)
    for s, t in enumerate(sets):
        one = pb.attr_lift_encode(glp, qs[s], xyz, t.attrs, lcp_enabled=t.lcp, bitdepth=t.bits)
        assert_results_equal([got[s]], [one], f"set {s}")
        assert np.array_equal(dec[s], one[1]), s
    assert got[0][2].any()  # the colour set did use last-component prediction


def batch_units(seed=3):
    """four units of different sizes (one of 48 points), each with its own dist2"""
    units = []
    for i, (n, dist2) in enumerate(((60000, 0), (48, 3), (25000, 7), (9000, 12))):
        xyz, rgb = cloud_shell(n, bits=9 if n > 1000 else 6, seed=seed + i)
        xyz = np.ascontiguousarray(xyz[:n])
        rgb = np.ascontiguousarray(texture(rgb[:n], 16, 50 + i).astype(np.int32))
        units.append((make_lod_params(levels=8, dist2=dist2), xyz, colour_and_refl(rgb, 16, 60 + i)))
    assert units[1][1].shape[0] == 48
    return units


def _run_batch(pb, units, forward=True, data=None, lcps=None):
    sets = units[0][2]
    lods = [_pods(u[0], sets)[0] for u in units]
    qs = _pods(units[0][0], sets)[1]
    if data is None:
        data = [[s.attrs for s in u[2]] for u in units]
    return pb.attr_lift_multi_batch(forward, lods, qs, [u[1] for u in units], data,
                                    [s.lcp for s in sets], [s.bits for s in sets], lcps)


@pytest.mark.gpu
def test_gpu_batch():
    import torch

    import pcc_attr_b200 as pb

    units = batch_units()
    vals, recs, lcps = _run_batch(pb, units)
    for i, (lp, xyz, sets) in enumerate(units):
        one, _ = _gpu_multi(lp, xyz, sets)
        assert_results_equal(list(zip(vals[i], recs[i], lcps[i])), one, f"unit {i}")
    dec = _run_batch(pb, units, False, vals, lcps)
    for i in range(len(units)):
        for s in range(2):
            assert np.array_equal(dec[i][s], recs[i][s]), (i, s)

    sets = units[0][2]
    lods = [_pods(u[0], sets)[0] for u in units]
    qs = _pods(units[0][0], sets)[1]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dx = [T(u[1]) for u in units]
    da = [[T(s.attrs) for s in u[2]] for u in units]
    dv = [[torch.zeros_like(a) for a in u] for u in da]
    rows = np.zeros((len(units), 2, MAX_LODS), dtype=np.int8)
    torch.cuda.synchronize()
    en, bd = [s.lcp for s in sets], [s.bits for s in sets]
    pb.attr_lift_multi_batch_dev(True, lods, qs, dx, da, dv, rows, en, bd)
    for i, lp in enumerate(lods):
        for s in range(2):
            assert np.array_equal(dv[i][s].cpu().numpy(), vals[i][s]), (i, s)
            assert np.array_equal(da[i][s].cpu().numpy(), recs[i][s]), (i, s)
            assert np.array_equal(rows[i, s, :lp.num_detail_levels], lcps[i][s]), (i, s)
    dd = [[torch.zeros_like(a) for a in u] for u in da]
    pb.attr_lift_multi_batch_dev(False, lods, qs, dx, dd, dv, rows, en, bd)
    for i in range(len(units)):
        for s in range(2):
            assert np.array_equal(dd[i][s].cpu().numpy(), recs[i][s]), (i, s)


@pytest.mark.gpu
def test_gpu_launches_do_not_scale_with_lifting_passes():
    import pcc_attr_b200 as pb

    xyz, rgb = cloud_shell(50000, bits=10, seed=4)
    rgb = np.ascontiguousarray(texture(rgb, 16, 5).astype(np.int32))
    both = colour_and_refl(rgb, 16)

    def launches(fn):
        before = pb.kernel_launch_count()
        fn()
        return pb.kernel_launch_count() - before

    extra = {}
    for levels in (4, 12):
        lp = make_lod_params(levels=levels)
        glp, qs = _pods(lp, both)
        multi = lambda sets: pb.attr_lift_multi_encode(glp, qs[:len(sets)], xyz, [s.attrs for s in sets],
                                                       [s.lcp for s in sets], [s.bits for s in sets])
        multi(both)  # warm-up
        one = launches(lambda: multi(both[:1]))
        two = launches(lambda: multi(both))
        refl = launches(lambda: pb.attr_lift_encode(glp, qs[1], xyz, both[1].attrs, 1, 16))
        assert one == launches(lambda: pb.attr_lift_encode(glp, qs[0], xyz, rgb, 1, 8)), levels
        extra[levels] = two - one
        assert 0 < extra[levels] < refl, (levels, one, two, refl)
    assert extra[4] == extra[12], extra


@pytest.mark.gpu
def test_gpu_concurrent_batches():
    """two host threads calling _multi_batch at once get what sequential calls get"""
    import pcc_attr_b200 as pb

    jobs = [batch_units(seed=3), batch_units(seed=9)]
    seq = [_run_batch(pb, u) for u in jobs]
    got, errors = [None, None], []

    def work(j):
        try:
            got[j] = _run_batch(pb, jobs[j])
        except Exception as e:  # reported below
            errors.append(e)

    ts = [threading.Thread(target=work, args=(j,)) for j in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for j in range(2):
        for part in range(3):
            for i in range(len(jobs[j])):
                for s in range(2):
                    assert np.array_equal(got[j][part][i][s], seq[j][part][i][s]), (j, part, i, s)


@pytest.mark.gpu
def test_gpu_own_level_predictors_unsupported():
    import pcc_attr_b200 as pb

    xyz, rgb = cloud_shell(5000, bits=8, seed=6)
    rgb = np.ascontiguousarray(rgb.astype(np.int32))
    lp = make_lod_params(decimation=0, skip_layers=0, intra_range=128, inter_range=128)
    sets = colour_and_refl(rgb, 8)
    glp, qs = _pods(lp, sets)
    lib = pb.lib()
    vals = np.zeros_like(rgb)
    rec = rgb.copy()
    rc = lib.pccb200_attr_lift_encode(C.byref(glp), C.byref(qs[0]), C.c_int32(1), None, _ptr(xyz, C.c_int32),
                                      _ptr(rec, C.c_int32), C.c_int32(3), C.c_int32(xyz.shape[0]), C.c_int32(8),
                                      _ptr(vals, C.c_int32), None)
    assert rc == UNSUPPORTED
    with pytest.raises(pb.PccB200Error, match="status 5"):
        pb.attr_lift_multi_encode(glp, qs, xyz, [s.attrs for s in sets], [1, 1], [8, 8])
