"""Recolouring several attribute sets on the same positions in one pass, and
many slices or frames per call (pccb200_recolour_multi, _multi_dev,
_multi_batch, _multi_batch_dev).  Every set's output must be bit-identical to
the one-set path and so to the oracle run once per set: on the host through
the product's kernel bodies (tests/emu), and -- on a GPU -- through the C ABI."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from pcc_testlib import ROOT, _ptr, coded_geometry, make_recolour_params, oracle_recolour
from pcc_attr_b200.synth import cloud_shell, texture

INVALID = 1  # PCCB200_ERR_INVALID_ARG

CASES = {
    # name: (scale, offset, params); colour and reflectance on the same positions
    "colour_half": (0.5, (0, 0, 0), {}),
    "colour_same": (1.0, (0, 0, 0), {}),
    "colour_offset": (0.37, (5, 3, 9), dict(search_range=2)),
    "refl_half": (0.5, (0, 0, 0), {}),
    "refl_k": (0.25, (0, 0, 0), dict(num_neighbours_fwd=5, num_neighbours_bwd=2)),
    "plain_avg": (0.5, (0, 0, 0), dict(use_dist_weighted_avg_fwd=0, use_dist_weighted_avg_bwd=0,
                                        skip_avg_if_identical_source_point_present_bwd=1)),
    "attr_prune": (0.5, (0, 0, 0), dict(max_attribute_dist2_fwd=300., max_attribute_dist2_bwd=200.)),
    "geom_limit": (0.5, (0, 0, 0), dict(max_geometry_dist2_fwd=6., max_geometry_dist2_bwd=3.)),
}


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


def make_case(name, n=6000, bits=8, seed=11, refl_bits=8):
    scale, off, kw = CASES[name]
    xyz, rgb = cloud_shell(n, bits=bits, seed=seed)
    rgb = texture(rgb, 20, seed + 1)
    refl = reflectance(rgb, refl_bits, seed + 2)
    tgt = coded_geometry(xyz, scale) - np.array(off, dtype=np.int32)
    tgt = np.ascontiguousarray(tgt[(tgt >= 0).all(axis=1)])
    return xyz, [rgb, refl], [8, refl_bits], scale, off, tgt, make_recolour_params(**kw)


_emu = None


def load_emu_multi():
    """tests/emu/emu_recolour_multi.cpp built for the host (once per process, in
    a temporary directory)"""
    global _emu
    if _emu is None:
        emu_dir = os.path.join(ROOT, "tests", "emu")
        tmp = tempfile.mkdtemp(prefix="emu_recolour_multi_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libemu_recolour_multi.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unused-variable",
                               "-x", "c++", "-I" + os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "csrc"),
                               "-I" + os.path.join(ROOT, "include"), "-I" + emu_dir,
                               os.path.join(emu_dir, "emu_recolour_multi.cpp"), "-o", so])
        _emu = C.CDLL(so)
    return _emu


def emu_recolour_multi(params, sxyz, attrs, bitdepths, scale, off, txyz):
    """the fused kernel bodies on the host: -> outs[s]"""
    lib = load_emu_multi()
    sxyz = np.ascontiguousarray(sxyz, dtype=np.int32)
    txyz = np.ascontiguousarray(txyz, dtype=np.int32)
    attrs = [np.ascontiguousarray(a, dtype=np.int32).reshape(sxyz.shape[0], -1) for a in attrs]
    k = len(attrs)
    outs = [np.zeros((txyz.shape[0], a.shape[1]), dtype=np.int32) for a in attrs]
    IP = C.POINTER(C.c_int32) * k
    o = np.ascontiguousarray(off, dtype=np.int32)
    rc = lib.emu_recolour_multi(C.byref(params), C.c_int(k), _ptr(sxyz, C.c_int32), C.c_int(sxyz.shape[0]),
                                IP(*[_ptr(a, C.c_int32) for a in attrs]),
                                (C.c_int32 * k)(*[a.shape[1] for a in attrs]), (C.c_int32 * k)(*bitdepths),
                                C.c_double(scale), _ptr(o, C.c_int32), _ptr(txyz, C.c_int32),
                                C.c_int(txyz.shape[0]), IP(*[_ptr(x, C.c_int32) for x in outs]))
    assert rc == 0, rc
    return outs


def oracle_per_set(params, sxyz, attrs, bitdepths, scale, off, txyz):
    return [oracle_recolour(params, sxyz, a, scale, off, txyz, bitdepth=b) for a, b in zip(attrs, bitdepths)]


def assert_sets_equal(got, exp, what):
    assert len(got) == len(exp)
    for s, (g, e) in enumerate(zip(got, exp)):
        assert g.shape == e.shape, (what, s, g.shape, e.shape)
        assert np.array_equal(g, e), (what, s, int((g != e).any(axis=1).sum()))


# ---- host: the fused kernel bodies against the oracle -------------------------

@pytest.mark.parametrize("refl_bits", [8, 16])
@pytest.mark.parametrize("name", list(CASES))
def test_emu_multi_vs_oracle(name, refl_bits):
    sx, attrs, bds, scale, off, tx, p = make_case(name, refl_bits=refl_bits)
    assert_sets_equal(emu_recolour_multi(p, sx, attrs, bds, scale, off, tx),
                      oracle_per_set(p, sx, attrs, bds, scale, off, tx), name)


@pytest.mark.parametrize("num_sets", [3, 4])
def test_emu_three_and_four_sets(num_sets):
    sx, (rgb, refl8), _, scale, off, tx, p = make_case("colour_offset", seed=5)
    refl16 = reflectance(rgb, 16, 9)
    rgb10 = np.ascontiguousarray(np.clip(rgb * 4 + 3, 0, 1023))
    attrs = [rgb, refl16, refl8, rgb10][:num_sets]
    bds = [8, 16, 8, 10][:num_sets]
    assert_sets_equal(emu_recolour_multi(p, sx, attrs, bds, scale, off, tx),
                      oracle_per_set(p, sx, attrs, bds, scale, off, tx), num_sets)


def test_emu_swapped_set_order():
    sx, attrs, bds, scale, off, tx, p = make_case("refl_k", refl_bits=16)
    fwd = emu_recolour_multi(p, sx, attrs, bds, scale, off, tx)
    rev = emu_recolour_multi(p, sx, attrs[::-1], bds[::-1], scale, off, tx)
    assert_sets_equal(rev, fwd[::-1], "swapped")


@pytest.mark.parametrize("seed", range(12))
def test_emu_multi_fuzz(seed):
    """parameters, scales, offsets and cloud shapes drawn as in
    test_recolour.py::test_kernel_bodies_fuzz; two sets, one of each width"""
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(200, 3000))
    if seed % 3 == 0:
        sx = np.unique(rng.integers(0, int(rng.integers(8, 3000)), size=(n, 3)).astype(np.int32), axis=0)
    else:
        sx, _ = cloud_shell(n, bits=int(rng.integers(5, 10)), seed=seed)
    if seed % 4 == 1:  # a few outliers far away from everything
        sx = np.concatenate([sx, rng.integers(100000, 2000000, size=(5, 3)).astype(np.int32)])
    a = 3 if seed % 2 else 1
    sa = rng.integers(0, 1 << 8, size=(sx.shape[0], a)).astype(np.int32)
    scale = float(rng.choice([1.0, 0.5, 0.25, 0.731, 1.37, 2.0]))
    off = tuple(int(v) for v in rng.integers(0, 7, size=3))
    tx = coded_geometry(sx, scale) - np.array(off, dtype=np.int32)
    tx = np.ascontiguousarray(tx[(tx >= 0).all(axis=1) & (tx < (1 << 21)).all(axis=1)])
    if tx.shape[0] < 20:
        pytest.skip("degenerate target")
    kf = int(rng.integers(1, min(16, sx.shape[0]) + 1))
    kb = int(rng.integers(1, min(4, tx.shape[0]) + 1))
    p = make_recolour_params(
        num_neighbours_fwd=kf, num_neighbours_bwd=kb, search_range=int(rng.integers(0, 3)),
        use_dist_weighted_avg_fwd=int(rng.integers(0, 2)), use_dist_weighted_avg_bwd=int(rng.integers(0, 2)),
        skip_avg_if_identical_source_point_present_fwd=int(rng.integers(0, 2)),
        skip_avg_if_identical_source_point_present_bwd=int(rng.integers(0, 2)),
        max_geometry_dist2_fwd=float(rng.choice([1000., 50., 4.])),
        max_geometry_dist2_bwd=float(rng.choice([1000., 9., 2.])),
        max_attribute_dist2_fwd=float(rng.choice([1000., 400., 60.])),
        max_attribute_dist2_bwd=float(rng.choice([1000., 300.])),
        dist_offset_fwd=float(rng.choice([4., 1., 0.5])), dist_offset_bwd=float(rng.choice([4., 2.])))
    bd2 = int(rng.choice([8, 10, 12, 16]))
    sa2 = rng.integers(0, 1 << bd2, size=(sx.shape[0], 4 - a)).astype(np.int32)
    attrs, bds = [sa, sa2], [8, bd2]
    assert_sets_equal(emu_recolour_multi(p, sx, attrs, bds, scale, off, tx),
                      oracle_per_set(p, sx, attrs, bds, scale, off, tx), seed)


# ---- the C entries refuse malformed arguments before they look for a device ----

class _Call:
    """one well-formed call of each new entry (host arrays; the *_dev entries are
    never given a device here, so their pointers are not dereferenced)"""

    def __init__(self):
        import pcc_attr_b200 as pb

        self.lib = pb.lib()
        self.p = pb.default_recolour_params()
        self.sx = [np.zeros((16, 3), dtype=np.int32), np.zeros((12, 3), dtype=np.int32)]
        self.tx = [np.zeros((10, 3), dtype=np.int32), np.zeros((9, 3), dtype=np.int32)]
        self.sa = [[np.zeros((16, 3), dtype=np.int32), np.zeros((16, 1), dtype=np.int32)],
                   [np.zeros((12, 3), dtype=np.int32), np.zeros((12, 1), dtype=np.int32)]]
        self.out = [[np.zeros((10, 3), dtype=np.int32), np.zeros((10, 1), dtype=np.int32)],
                    [np.zeros((9, 3), dtype=np.int32), np.zeros((9, 1), dtype=np.int32)]]

    def args(self, **kw):
        """C arguments of a two-unit, two-set batch call; kw overrides any of them"""
        a = dict(params=C.byref(self.p), num_sets=2, num_units=2,
                 sx=[x.ctypes.data for x in self.sx], ns=[16, 12],
                 sa=[a.ctypes.data for u in self.sa for a in u], na=[3, 1], bd=[8, 16],
                 scale=[1.0, 0.5], off=[0, 0, 0, 1, 2, 3], tx=[x.ctypes.data for x in self.tx],
                 nt=[10, 9], out=[o.ctypes.data for u in self.out for o in u])
        a.update(kw)
        return a

    @staticmethod
    def _arr(t, v):
        return None if v is None else (t * len(v))(*v)

    def batch(self, dev=False, **kw):
        a = self.args(**kw)
        fn = self.lib.pccb200_recolour_multi_batch_dev if dev else self.lib.pccb200_recolour_multi_batch
        A = self._arr
        return fn(a["params"], C.c_int32(a["num_sets"]), C.c_int32(a["num_units"]), A(C.c_void_p, a["sx"]),
                  A(C.c_int32, a["ns"]), A(C.c_void_p, a["sa"]), A(C.c_int32, a["na"]), A(C.c_int32, a["bd"]),
                  A(C.c_double, a["scale"]), A(C.c_int32, a["off"]), A(C.c_void_p, a["tx"]),
                  A(C.c_int32, a["nt"]), A(C.c_void_p, a["out"]))

    def single(self, dev=False, **kw):
        """unit 0 of args() through pccb200_recolour_multi(_dev)"""
        a = self.args(**kw)
        fn = self.lib.pccb200_recolour_multi_dev if dev else self.lib.pccb200_recolour_multi
        A = self._arr
        k = a["num_sets"]
        return fn(a["params"], C.c_int32(k), C.c_void_p(a["sx"][0]) if a["sx"] else None,
                  C.c_int32(a["ns"][0]), A(C.c_void_p, a["sa"][:k] if a["sa"] else None),
                  A(C.c_int32, a["na"]), A(C.c_int32, a["bd"]), C.c_double(a["scale"][0]),
                  A(C.c_int32, a["off"][:3] if a["off"] else None),
                  C.c_void_p(a["tx"][0]) if a["tx"] else None, C.c_int32(a["nt"][0]),
                  A(C.c_void_p, a["out"][:k] if a["out"] else None))


def _malformed(c):
    """(what, overrides) for every kind of malformed input"""
    import pcc_attr_b200 as pb

    def params(**kw):
        p = pb.default_recolour_params()
        for k, v in kw.items():
            setattr(p, k, v)
        c.keep = getattr(c, "keep", []) + [p]
        return C.byref(p)

    sx, sa, out, tx = c.args()["sx"], c.args()["sa"], c.args()["out"], c.args()["tx"]
    return [
        ("null params", dict(params=None)),
        ("null source positions", dict(sx=None)),
        ("null source positions of a unit", dict(sx=[sx[0], None])),
        ("null target positions", dict(tx=None)),
        ("null target positions of a unit", dict(tx=[None, tx[1]])),
        ("null attribute array", dict(sa=None)),
        ("null source attributes of a set", dict(sa=[sa[0], None, sa[2], sa[3]])),
        ("null output array", dict(out=None)),
        ("null output of a set", dict(out=[None, out[1], out[2], out[3]])),
        ("null component counts", dict(na=None)),
        ("null bit depths", dict(bd=None)),
        ("null scales", dict(scale=None)),
        ("null offsets", dict(off=None)),
        ("null point counts", dict(ns=None)),
        ("num_sets 0", dict(num_sets=0)),
        ("num_sets 5", dict(num_sets=5, na=[3, 1, 1, 1, 1], bd=[8] * 5, sa=sa * 3, out=out * 3)),
        ("two components", dict(na=[3, 2])),
        ("four components", dict(na=[4, 1])),
        ("bit depth 0", dict(bd=[0, 8])),
        ("bit depth 17", dict(bd=[8, 17])),
        ("no source points", dict(ns=[16, 0])),
        ("negative target count", dict(nt=[-1, 9])),
        ("forward neighbours above 16", dict(params=params(num_neighbours_fwd=17))),
        ("forward neighbours above the source points", dict(ns=[7, 12])),
        ("no forward neighbours", dict(params=params(num_neighbours_fwd=0))),
        ("backward neighbours above 16", dict(params=params(num_neighbours_bwd=17))),
        ("backward neighbours above the target points", dict(params=params(num_neighbours_bwd=11))),
        ("search range -1", dict(params=params(search_range=-1))),
        ("search range 9", dict(params=params(search_range=9))),
        ("scale 0", dict(scale=[1.0, 0.0])),
        ("negative scale", dict(scale=[-0.5, 1.0])),
        ("NaN scale", dict(scale=[float("nan"), 1.0])),
    ]


@pytest.mark.parametrize("dev", [False, True])
def test_batch_entry_argument_checks(dev):
    import torch

    c = _Call()
    for what, kw in _malformed(c) + [("no units", dict(num_units=0))]:
        assert c.batch(dev, **kw) == INVALID, what
    if not torch.cuda.is_available():
        rc = c.batch(dev)
        assert rc not in (0, INVALID)
        assert b"CUDA" in c.lib.pccb200_last_error() or b"device" in c.lib.pccb200_last_error()


@pytest.mark.parametrize("dev", [False, True])
def test_single_entry_argument_checks(dev):
    """pccb200_recolour_multi(_dev): unit 0 of the same cases (a case that only
    breaks unit 1 is well-formed here)"""
    import torch

    c = _Call()
    for what, kw in _malformed(c):
        if "of a unit" in what or what in ("null point counts", "null scales"):
            continue
        kw = {"no source points": dict(ns=[0]), "scale 0": dict(scale=[0.0])}.get(what, kw)
        assert c.single(dev, **kw) == INVALID, what
    if not torch.cuda.is_available():
        rc = c.single(dev)
        assert rc not in (0, INVALID)
        assert b"CUDA" in c.lib.pccb200_last_error() or b"device" in c.lib.pccb200_last_error()


# ---- GPU: the C entries against the oracle and against the one-set call ---------

def _pp(p):
    import pcc_attr_b200 as pb

    return pb.RecolourParams.from_buffer_copy(bytes(p))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_multi_vs_oracle(name):
    import pcc_attr_b200 as pb

    sx, attrs, bds, scale, off, tx, p = make_case(name, n=30000, bits=9, seed=21, refl_bits=16)
    g = pb.recolour_multi(_pp(p), sx, attrs, tx, scale, off, bds)
    assert_sets_equal(g, oracle_per_set(p, sx, attrs, bds, scale, off, tx), name)


@pytest.mark.gpu
def test_gpu_multi_full_size():
    """1M-point 11-bit source, colour + 16-bit reflectance at scale 0.5: equal to
    two pccb200_recolour calls and to the fused kernel bodies on the host"""
    import pcc_attr_b200 as pb

    xyz, rgb = cloud_shell(1000000, bits=11, seed=7)
    rgb = texture(rgb, 16, 8)
    refl = reflectance(rgb, 16, 9)
    tx = coded_geometry(xyz, 0.5)
    p = make_recolour_params()
    g = pb.recolour_multi(_pp(p), xyz, [rgb, refl], tx, 0.5, (0, 0, 0), [8, 16])
    one = [pb.recolour(_pp(p), xyz, rgb, tx, 0.5, bitdepth=8), pb.recolour(_pp(p), xyz, refl, tx, 0.5, bitdepth=16)]
    assert_sets_equal(g, one, "two pccb200_recolour calls")
    assert_sets_equal(g, emu_recolour_multi(p, xyz, [rgb, refl], [8, 16], 0.5, (0, 0, 0), tx), "emu")


def batch_units(seed=3):
    """about 24 units: four slices of one frame (each relative to its own origin,
    different offsets), frames at scales 1.0, 0.5 and 0.37 from 200k points
    down, and the smallest legal unit (8 source points, 1 target point)"""
    units = []
    xyz, rgb = cloud_shell(120000, bits=10, seed=seed)
    rgb = texture(rgb, 20, seed + 1)
    order = np.argsort(xyz[:, 0], kind="stable")
    for i, part in enumerate(np.array_split(order, 4)):
        sx = xyz[part]
        origin = sx.min(axis=0)
        sx = np.ascontiguousarray(sx - origin)
        off = (i, 2 * i % 5, 3)
        tx = coded_geometry(sx, 0.5) - np.array(off, dtype=np.int32)
        tx = np.ascontiguousarray(tx[(tx >= 0).all(axis=1)])
        units.append((sx, [np.ascontiguousarray(rgb[part]), reflectance(rgb[part], 16, 40 + i)], tx, 0.5, off))
    sizes = [200000, 90000, 40000, 20000, 9000, 5000, 2000, 1000, 400, 100, 60, 30]
    scales = [1.0, 0.5, 0.37]
    for i, n in enumerate(sizes + sizes[::3]):
        sx, c = cloud_shell(n, bits=int(8 + (n > 5000) + (n > 50000)), seed=100 + i)
        c = texture(c, 12, 200 + i)
        scale = scales[i % 3]
        off = (i % 3, 0, i % 2)
        tx = coded_geometry(sx, scale) - np.array(off, dtype=np.int32)
        tx = np.ascontiguousarray(tx[(tx >= 0).all(axis=1)])
        units.append((sx, [c, reflectance(c, 16, 300 + i)], tx, scale, off))
    rng = np.random.default_rng(seed)
    sx = np.unique(rng.integers(0, 50, size=(40, 3)).astype(np.int32), axis=0)[:8]
    units.append((np.ascontiguousarray(sx), [rng.integers(0, 256, size=(8, 3)).astype(np.int32),
                                            rng.integers(0, 65536, size=(8, 1)).astype(np.int32)],
                  np.ascontiguousarray(sx[:1] // 2), 0.5, (0, 0, 0)))
    return units


def _run_batch(pb, p, units):
    return pb.recolour_multi_batch(p, [u[0] for u in units], [u[1] for u in units], [u[2] for u in units],
                                   [u[3] for u in units], [u[4] for u in units], [8, 16])


@pytest.mark.gpu
def test_gpu_batch():
    import torch

    import pcc_attr_b200 as pb

    units = batch_units()
    assert 20 <= len(units) <= 28
    assert max(u[0].shape[0] for u in units) == 200000
    p = _pp(make_recolour_params())
    host = _run_batch(pb, p, units)
    for i, (sx, attrs, tx, scale, off) in enumerate(units):
        one = [pb.recolour(p, sx, a, tx, scale, off, bitdepth=b) for a, b in zip(attrs, [8, 16])]
        assert_sets_equal(host[i], one, f"unit {i}")

    dev = torch.device("cuda")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dsx = [T(u[0]) for u in units]
    dtx = [T(u[2]) for u in units]
    dsa = [[T(a) for a in u[1]] for u in units]
    douts = [[torch.zeros((u[2].shape[0], a.shape[1]), dtype=torch.int32, device=dev) for a in u[1]]
             for u in units]
    torch.cuda.synchronize()
    pb.recolour_multi_batch_dev(p, dsx, dsa, dtx, [u[3] for u in units], [u[4] for u in units], douts, [8, 16])
    for i in range(len(units)):
        assert_sets_equal([o.cpu().numpy() for o in douts[i]], host[i], f"dev unit {i}")

    lib = pb.lib()
    for i in (0, len(units) // 2, len(units) - 1):
        outs = [torch.zeros_like(o) for o in douts[i]]
        VP = C.c_void_p * 2
        rc = lib.pccb200_recolour_multi_dev(
            C.byref(p), C.c_int32(2), C.c_void_p(dsx[i].data_ptr()), C.c_int32(units[i][0].shape[0]),
            VP(*[a.data_ptr() for a in dsa[i]]), (C.c_int32 * 2)(3, 1), (C.c_int32 * 2)(8, 16),
            C.c_double(units[i][3]), (C.c_int32 * 3)(*units[i][4]), C.c_void_p(dtx[i].data_ptr()),
            C.c_int32(units[i][2].shape[0]), VP(*[o.data_ptr() for o in outs]))
        assert rc == 0, lib.pccb200_last_error()
        assert_sets_equal([o.cpu().numpy() for o in outs], host[i], f"multi_dev unit {i}")


@pytest.mark.gpu
def test_gpu_bad_coordinate_names_the_unit():
    """a coordinate outside [0, 2^21) is only found on the device"""
    import pcc_attr_b200 as pb

    units = batch_units()[:6]
    sx = units[4][0].copy()
    sx[3, 1] = 1 << 21
    units[4] = (sx,) + units[4][1:]
    with pytest.raises(pb.PccB200Error, match="unit 4"):
        _run_batch(pb, _pp(make_recolour_params()), units)


@pytest.mark.gpu
def test_gpu_launches_do_not_depend_on_sets():
    import pcc_attr_b200 as pb

    sx, attrs, bds, scale, off, tx, p = make_case("colour_half", n=50000, bits=10, seed=4, refl_bits=16)
    p = _pp(p)
    pb.recolour_multi(p, sx, attrs[:1], tx, scale, off, bds[:1])  # warm-up

    def launches(fn):
        before = pb.kernel_launch_count()
        fn()
        return pb.kernel_launch_count() - before

    one = launches(lambda: pb.recolour_multi(p, sx, attrs[:1], tx, scale, off, bds[:1]))
    two = launches(lambda: pb.recolour_multi(p, sx, attrs, tx, scale, off, bds))
    four = launches(lambda: pb.recolour_multi(p, sx, attrs + attrs, tx, scale, off, bds + bds))
    legacy = launches(lambda: pb.recolour(p, sx, attrs[0], tx, scale, off))
    assert one > 0 and one == two == four == legacy, (one, two, four, legacy)


@pytest.mark.gpu
def test_gpu_concurrent_batches():
    """four host threads calling _multi_batch at once on different inputs get
    what sequential calls get"""
    import pcc_attr_b200 as pb

    p = _pp(make_recolour_params())
    jobs = []
    for j in range(4):
        units = []
        for i in range(5):
            sx, c = cloud_shell(20000 + 7000 * i, bits=9, seed=500 + 10 * j + i)
            c = texture(c, 16, 600 + 10 * j + i)
            scale = [1.0, 0.5, 0.37][(i + j) % 3]
            units.append((sx, [c, reflectance(c, 16, j * 10 + i)], coded_geometry(sx, scale), scale, (0, 0, 0)))
        jobs.append(units)
    seq = [_run_batch(pb, p, u) for u in jobs]
    got = [None] * 4
    errors = []

    def work(j):
        try:
            got[j] = _run_batch(pb, p, jobs[j])
        except Exception as e:  # reported below
            errors.append(e)

    ts = [threading.Thread(target=work, args=(j,)) for j in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for j in range(4):
        for i in range(len(jobs[j])):
            assert_sets_equal(got[j][i], seq[j][i], f"thread {j} unit {i}")
