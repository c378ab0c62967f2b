"""Reference-exact recolouring (pccb200_recolour_exact, _exact_multi_batch,
_exact_multi_batch_dev): nanoflann's kd-tree built level by level, its
findNeighbors, and libstdc++'s std::sort order of the backward lists.

On the CPU the product's kernel bodies run through tests/emu and are compared
with the reference: the tree (vind, leaf ranges, divfeat, divlow / divhigh),
the k-nearest-neighbour lists element for element, the std::sort restatement
and the recolouring itself.  The reference is oracle/_ref/libtmc13_kdtree.so and
libtmc13_recolour.so where they are built; elsewhere the SHA-256 digests of
its results, recorded in tests/golden/recolour_exact_golden.npz by
tests/golden/make_recolour_exact_golden.py, stand in for them.  On a GPU the three
entries are compared with the same results, with one-unit calls and with the
emulation, and the whole encoder with the recolouring drop-in against the
unmodified one."""
import atexit
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from pcc_testlib import (ORACLE_DIR, ROOT, _ptr, coded_geometry, make_recolour_params, ref_recolour,
                         results_digest)
from pcc_attr_b200.synth import cloud_shell, texture
from test_recolour import CASES as RECOLOUR_CASES, _case as recolour_case

GOLDEN = os.path.join(ROOT, "tests", "golden", "recolour_exact_golden.npz")
KDTREE_SO = os.path.join(ORACLE_DIR, "_ref", "libtmc13_kdtree.so")
RECOLOUR_SO = os.path.join(ORACLE_DIR, "_ref", "libtmc13_recolour.so")


def live():
    """the compiled reference (oracle/_ref) is present"""
    return os.path.exists(KDTREE_SO) and os.path.exists(RECOLOUR_SO)


_golden = None


def recorded_digest(key):
    """the recorded digest of the reference's results for `key`"""
    global _golden
    if _golden is None:
        g = np.load(GOLDEN)
        _golden = dict(zip(g["keys"].tolist(), g["digests"]))
    assert key in _golden, f"no recorded result for {key} (tests/golden/make_recolour_exact_golden.py)"
    return _golden[key]


def matches_reference(key, got):
    """got (a list of arrays) equals the reference's results for `key`"""
    if live():
        exp = golden_entries()[key]()
        return len(exp) == len(got) and all(np.array_equal(e, g) for e, g in zip(exp, got))
    return np.array_equal(results_digest(got), recorded_digest(key))


def check_reference(key, got, labels=None):
    """assert that got (a list of arrays) equals the reference's results for
    `key`: element by element where the reference is built, else by digest"""
    if live():
        exp = golden_entries()[key]()
        assert len(exp) == len(got), key
        for i, (e, g) in enumerate(zip(exp, got)):
            e, g = np.asarray(e), np.asarray(g)
            what = labels[i] if labels else i
            assert e.shape == g.shape and np.array_equal(e, g), (
                key, what, int((e != g).reshape(e.shape[0], -1).any(axis=1).sum()) if e.shape == g.shape else None)
    else:
        assert np.array_equal(results_digest(got), recorded_digest(key)), f"{key}: differs from the reference"


# ---- libraries ----------------------------------------------------------------

_emu = None
_kd = None


def load_emu_exact():
    """tests/emu/emu_recolour_exact.cpp built for the host (once per process,
    in a temporary directory)"""
    global _emu
    if _emu is None:
        emu_dir = os.path.join(ROOT, "tests", "emu")
        tmp = tempfile.mkdtemp(prefix="emu_recolour_exact_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libemu_recolour_exact.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unused-variable",
                               "-x", "c++", "-I" + os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "csrc"),
                               "-I" + os.path.join(ROOT, "include"), "-I" + emu_dir,
                               os.path.join(emu_dir, "emu_recolour_exact.cpp"), "-o", so])
        _emu = C.CDLL(so)
        _emu.emu_gnu_sort.restype = None
    return _emu


def load_kd():
    global _kd
    if _kd is None:
        _kd = C.CDLL(KDTREE_SO)
        _kd.ref_std_sort.restype = None
    return _kd


def _tree(fn, xyz):
    n = xyz.shape[0]
    vind = np.zeros(n, np.int32)
    info = np.zeros((2 * n, 4), np.int32)
    div = np.zeros((2 * n, 2))
    box = np.zeros(6)
    depth = np.zeros(1, np.int32)
    m = fn(_ptr(xyz, C.c_int32), n, _ptr(vind, C.c_int32), _ptr(info, C.c_int32), _ptr(div, C.c_double),
           _ptr(box, C.c_double), _ptr(depth, C.c_int32))
    assert m > 0
    return [vind, info[:m].copy(), div[:m].copy(), box, depth]


def _knn(fn, xyz, q, k):
    idx = np.zeros((q.shape[0], k), np.int32)
    dist = np.zeros((q.shape[0], k))
    assert fn(_ptr(xyz, C.c_int32), xyz.shape[0], _ptr(q, C.c_double), q.shape[0], k,
              _ptr(idx, C.c_int32), _ptr(dist, C.c_double)) == 0
    return [idx, dist]


def _sort(fn, key, val):
    key, val = key.copy(), val.copy()
    fn(_ptr(key, C.c_double), _ptr(val, C.c_int32), key.shape[0])
    return [key, val]


def _recolour(fn, p, sx, sa, scale, off, tx, bitdepth=8):
    sa = np.ascontiguousarray(sa, dtype=np.int32)
    a = sa.shape[1]
    out = np.zeros((tx.shape[0], a), np.int32)
    o = np.ascontiguousarray(off, dtype=np.int32)
    rc = fn(C.byref(p), _ptr(sx, C.c_int32), _ptr(sa, C.c_int32), a, sx.shape[0], C.c_double(scale),
            _ptr(o, C.c_int32), _ptr(tx, C.c_int32), tx.shape[0], bitdepth, _ptr(out, C.c_int32))
    return rc, out


def emu_exact(p, sx, sa, scale, off, tx, bitdepth=8):
    rc, out = _recolour(load_emu_exact().emu_recolour_exact, p, sx, sa, scale, off, tx, bitdepth)
    assert rc == 0
    return out


def emu_grid(p, sx, sa, scale, off, tx, bitdepth=8):
    rc, out = _recolour(load_emu_exact().emu_recolour_grid, p, sx, sa, scale, off, tx, bitdepth)
    assert rc == 0
    return out


# ---- cases --------------------------------------------------------------------

def tree_clouds():
    rng = np.random.default_rng(3)
    shell, _ = cloud_shell(8000, bits=8, seed=3)
    dup = np.repeat(rng.integers(0, 6, size=(40, 3)), 25, axis=0)   # 25 copies of every point
    plane = np.c_[rng.integers(0, 200, size=(3000, 2)), np.full(3000, 7)]
    line = np.c_[np.full((2000, 2), -3), rng.integers(-500, 500, size=(2000, 1))]
    return {
        "shell": shell,
        "duplicates": np.concatenate([dup, np.repeat([[1, 2, 3]], 37, axis=0)]),
        "plane": plane,
        "line": line,
        "n1": np.array([[5, -4, 3]]),
        "n10": rng.integers(0, 3, size=(10, 3)),
        "n11": rng.integers(0, 3, size=(11, 3)),
        "negative": rng.integers(-(1 << 20), 1000, size=(4000, 3)),
        "big_range": np.concatenate([rng.integers(-(1 << 29), 1 << 29, size=(50, 3)),
                                     rng.integers(0, 64, size=(500, 3))]),
    }


def _cloud(name):
    return np.ascontiguousarray(tree_clouds()[name], dtype=np.int32)


KNN_SCALES = {1.0: (0, 0, 0), 0.5: (2, 0, 1), 0.37: (5, 3, 9), 0.25: (0, 4, 0)}


def knn_case(scale):
    """a voxelised shell and its coded geometry at `scale`: forward queries
    (target + offset) / scale in the source, backward source * scale - offset in
    the target, computed as recolour_run computes them"""
    off = KNN_SCALES[scale]
    src, _ = cloud_shell(3000, bits=8, seed=5)
    tgt = np.ascontiguousarray(coded_geometry(src, scale) - np.array(off, dtype=np.int32))
    o = np.array(off, dtype=np.float64)
    fwd = (tgt.astype(np.int64) + np.array(off)).astype(np.float64) * (1.0 / scale)
    bwd = src.astype(np.float64) * scale - o
    return src, tgt, np.ascontiguousarray(fwd[::2]), np.ascontiguousarray(bwd[::3])


def sort_lists():
    rng = np.random.default_rng(9)
    out = []
    for n in list(range(1, 70)) + [100, 257, 600, 1000, 2000]:
        for t in range(3):
            ties = max(1, n // (1 + 4 * t))
            key = rng.integers(0, ties, size=n).astype(np.float64) * 0.25
            out.append((key, np.arange(n, dtype=np.int32)))
    out.append((np.zeros(2000), np.arange(2000, dtype=np.int32)))                 # one value
    out.append((np.arange(2000, 0, -1).astype(np.float64), np.arange(2000, dtype=np.int32)))
    return out


# the recolouring cases: every case of test_recolour.py, plus one at scale 1/4
# whose backward lists exceed 16 entries (introsort's partition decides the
# order of equal distances there)
EXACT_CASES = list(RECOLOUR_CASES) + ["long_lists"]


def exact_case(name, n=6000, bits=8, seed=11):
    if name != "long_lists":
        return recolour_case(name, n, bits, seed)
    xyz, rgb = cloud_shell(n, bits=bits, seed=seed)
    rgb = texture(rgb, 20, seed + 1)
    tgt = np.ascontiguousarray(coded_geometry(xyz, 0.25))
    return xyz, rgb, 0.25, (0, 0, 0), tgt, make_recolour_params(num_neighbours_bwd=6, num_neighbours_fwd=12)


def golden_entries():
    """every recorded result: key -> function computing it with the live reference"""
    kd = load_kd() if live() else None
    e = {}
    for name in tree_clouds():
        e[f"tree/{name}"] = lambda name=name: _tree(kd.ref_kdtree_build, _cloud(name))
    for scale in KNN_SCALES:
        for k in (1, 2, 8, 16):
            def f(scale=scale, k=k):
                src, tgt, fq, bq = knn_case(scale)
                return _knn(kd.ref_kdtree_knn, src, fq, k) + _knn(kd.ref_kdtree_knn, tgt, bq, k)
            e[f"knn/{scale}/{k}"] = f
    e["sort"] = lambda: [_sort(kd.ref_std_sort, k, v)[1] for k, v in sort_lists()]
    for name in EXACT_CASES:
        def g(name=name):
            sx, sa, scale, off, tx, p = exact_case(name)
            return [ref_recolour(p, sx, sa, scale, off, tx)]
        e[f"recolour/{name}"] = g
    return e


# ---- CPU: the kernel bodies on the host against the reference ------------------

@pytest.mark.parametrize("name", list(tree_clouds()))
def test_tree_equals_nanoflann(name):
    """vind, the preorder node list (leaf ranges, divfeat, divlow, divhigh),
    the root box and the depth equal nanoflann's"""
    e = _tree(load_emu_exact().emu_kdtree_build, _cloud(name))
    check_reference(f"tree/{name}", e, ("vind", "nodes", "divlow/divhigh", "root box", "depth"))


@pytest.mark.parametrize("scale", list(KNN_SCALES))
@pytest.mark.parametrize("k", [1, 2, 8, 16])
def test_knn_equals_find_neighbours(scale, k):
    """forward and backward k-nearest lists equal findNeighbors element for
    element: indices, distances and their order"""
    src, tgt, fq, bq = knn_case(scale)
    emu = load_emu_exact()
    e = _knn(emu.emu_kdtree_knn, src, fq, k) + _knn(emu.emu_kdtree_knn, tgt, bq, k)
    check_reference(f"knn/{scale}/{k}", e, ("fwd idx", "fwd dist", "bwd idx", "bwd dist"))


def test_std_sort_restatement():
    """GnuSort on tie-heavy lists of 1 to 2000 entries leaves equal keys where
    the compiled std::sort does"""
    emu = load_emu_exact()
    got = []
    for key, val in sort_lists():
        k, v = _sort(emu.emu_gnu_sort, key, val)
        assert np.array_equal(k, np.sort(key))
        got.append(v)
    check_reference("sort", got, [f"list {i}, length {v.shape[0]}" for i, v in enumerate(got)])


@pytest.mark.parametrize("name", EXACT_CASES)
def test_emu_recolour_equals_reference(name):
    """the exact path's kernel bodies equal recolourColour / recolourReflectance
    bit for bit; at scales below 1 the lowest-index rule of the grid path gives a
    different result on the same case, so the case reaches distance ties"""
    sx, sa, scale, off, tx, p = exact_case(name)
    check_reference(f"recolour/{name}", [emu_exact(p, sx, sa, scale, off, tx)])
    if scale < 1:
        assert not matches_reference(f"recolour/{name}", [emu_grid(p, sx, sa, scale, off, tx)]), name


def test_long_lists_case_has_long_lists():
    """the long_lists case sends more than 16 sources to some targets"""
    from scipy.spatial import cKDTree

    sx, sa, scale, off, tx, p = exact_case("long_lists")
    _, idx = cKDTree(tx).query(sx * scale, k=p.num_neighbours_bwd)
    assert np.bincount(idx.ravel(), minlength=tx.shape[0]).max() > 16


def test_coordinate_range():
    """negative coordinates are accepted; |x| >= 2^30 (coordinate or offset) is refused"""
    xyz, rgb = cloud_shell(500, bits=6, seed=2)
    p = make_recolour_params()
    neg = xyz - 40
    fn = load_emu_exact().emu_recolour_exact
    assert _recolour(fn, p, neg, rgb, 1.0, (0, 0, 0), neg)[0] == 0
    assert np.array_equal(emu_exact(p, neg, rgb, 1.0, (0, 0, 0), neg), rgb)
    far = xyz.copy()
    far[3, 1] = 1 << 30
    assert _recolour(fn, p, far, rgb, 1.0, (0, 0, 0), xyz)[0] != 0
    assert _recolour(fn, p, xyz, rgb, 1.0, (0, 0, 0), far)[0] != 0
    assert _recolour(fn, p, xyz, rgb, 1.0, (0, -(1 << 30), 0), xyz)[0] != 0
    assert _recolour(fn, make_recolour_params(num_neighbours_fwd=17), xyz, rgb, 1.0, (0, 0, 0), xyz)[0] != 0


# ---- GPU ------------------------------------------------------------------------

def _pp(p):
    import pcc_attr_b200 as pb

    return pb.RecolourParams.from_buffer_copy(bytes(p))


@pytest.mark.gpu
@pytest.mark.parametrize("name", EXACT_CASES)
def test_gpu_entries_equal_reference(name):
    """the three entries equal the reference on every case"""
    import torch

    import pcc_attr_b200 as pb

    sx, sa, scale, off, tx, p = exact_case(name)
    key = f"recolour/{name}"
    pp = _pp(p)
    check_reference(key, [pb.recolour_exact(pp, sx, sa, tx, scale, off)])
    (b,), = pb.recolour_exact_multi_batch(pp, [sx], [[sa]], [tx], [scale], [off])
    check_reference(key, [b])
    dev = torch.device("cuda")
    out = torch.zeros(tx.shape[0], sa.shape[1], dtype=torch.int32, device=dev)
    pb.recolour_exact_multi_batch_dev(pp, [torch.from_numpy(sx).to(dev)], [[torch.from_numpy(sa).to(dev)]],
                                      [torch.from_numpy(tx).to(dev)], [scale], [off], [[out]])
    torch.cuda.synchronize()
    check_reference(key, [out.cpu().numpy()])


def bench_frame():
    """bench.py's recolouring workload: the 1M-point frame with RGB and 8-bit
    reflectance onto its half-resolution geometry"""
    xyz, rgb = cloud_shell(1000000, bits=11, seed=7)
    rgb = texture(rgb, 16, 8)
    refl = np.ascontiguousarray(((rgb[:, :1].astype(np.int64) * 2 + rgb[:, 1:2]) // 3).astype(np.int32))
    return xyz, rgb, refl, np.ascontiguousarray(coded_geometry(xyz, 0.5))


@pytest.mark.gpu
def test_gpu_bench_frame():
    """colour and reflectance of the 1M-point frame in one call equal two
    reference calls (or, without the compiled reference, the emulated bodies)"""
    import pcc_attr_b200 as pb

    xyz, rgb, refl, tx = bench_frame()
    p = make_recolour_params()
    col, rfl = pb.recolour_exact_multi_batch(_pp(p), [xyz], [[rgb, refl]], [tx], [0.5], [(0, 0, 0)])[0]
    want = ref_recolour if os.path.exists(RECOLOUR_SO) else emu_exact
    assert np.array_equal(col, want(p, xyz, rgb, 0.5, (0, 0, 0), tx))
    assert np.array_equal(rfl, want(p, xyz, refl, 0.5, (0, 0, 0), tx))


def batch_units(m=16):
    units = []
    for u in range(m):
        xyz, rgb = cloud_shell(3000 + 500 * u, bits=7 + u % 3, seed=40 + u)
        rgb = texture(rgb, 20, u)
        scale = [0.5, 0.37, 0.25, 1.0][u % 4]
        off = (u % 3, -(u % 5), 2) if u % 2 else (0, 0, 0)
        xyz = xyz - (20 * u)   # negative coordinates in later units
        tgt = np.ascontiguousarray(coded_geometry(xyz, scale) - np.array(off, dtype=np.int32))
        units.append((xyz.astype(np.int32), [rgb, np.ascontiguousarray(rgb[:, 1:2])], tgt, scale, off))
    return units


@pytest.mark.gpu
def test_gpu_batch_equals_unit_calls():
    """16 units in one call, host and device pointers, equal one-unit calls"""
    import torch

    import pcc_attr_b200 as pb

    p = _pp(make_recolour_params(num_neighbours_bwd=3))
    units = batch_units()
    per = [[pb.recolour_exact(p, x, a, t, s, o) for a in attrs] for x, attrs, t, s, o in units]
    got = pb.recolour_exact_multi_batch(p, [u[0] for u in units], [u[1] for u in units], [u[2] for u in units],
                                        [u[3] for u in units], [u[4] for u in units])
    dev = torch.device("cuda")
    outs = [[torch.zeros(t.shape[0], a.shape[1], dtype=torch.int32, device=dev) for a in attrs]
            for _, attrs, t, _, _ in units]
    pb.recolour_exact_multi_batch_dev(
        p, [torch.from_numpy(u[0]).to(dev) for u in units],
        [[torch.from_numpy(a).to(dev) for a in u[1]] for u in units],
        [torch.from_numpy(u[2]).to(dev) for u in units], [u[3] for u in units], [u[4] for u in units], outs)
    torch.cuda.synchronize()
    for i in range(len(units)):
        for s in range(2):
            assert np.array_equal(got[i][s], per[i][s]), (i, s)
            assert np.array_equal(outs[i][s].cpu().numpy(), per[i][s]), (i, s)


@pytest.mark.gpu
def test_gpu_concurrent_calls():
    """calls from several threads give the outputs of sequential calls"""
    import pcc_attr_b200 as pb

    p = _pp(make_recolour_params())
    units = batch_units(6)
    want = [pb.recolour_exact(p, x, attrs[0], t, s, o) for x, attrs, t, s, o in units]
    got = [None] * len(units)
    errors = []

    def run(i):
        try:
            x, attrs, t, s, o = units[i]
            for _ in range(3):
                got[i] = pb.recolour_exact(p, x, attrs[0], t, s, o)
                assert np.array_equal(got[i], want[i])
        except Exception as e:  # noqa: BLE001
            errors.append((i, e))

    threads = [threading.Thread(target=run, args=(i,)) for i in range(len(units))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


@pytest.mark.gpu
def test_gpu_grid_entries_unchanged():
    """the grid-hash entries still compute what the lowest-index oracle does
    on the test_recolour_multi inputs (their outputs are not changed by the
    second path)"""
    import pcc_attr_b200 as pb
    from pcc_testlib import oracle_recolour
    from test_recolour_multi import CASES as MULTI_CASES, make_case

    for name in MULTI_CASES:
        xyz, attrs, bits, scale, off, tgt, p = make_case(name, n=20000, bits=9, seed=21)
        outs = pb.recolour_multi(_pp(p), xyz, attrs, tgt, scale, off, bits)
        for a, b, o in zip(attrs, bits, outs):
            assert np.array_equal(o, oracle_recolour(p, xyz, a, scale, off, tgt, b)), name


# ---- whole codec ------------------------------------------------------------------

RECOLOUR_BIN = os.path.join(ORACLE_DIR, "_ref", "tmc3_b200_recolour")


def _write_ply(path, xyz, rgb, refl):
    with open(path, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
                "property uint16 refc\nend_header\n" % len(xyz))
        for p, c, r in zip(xyz, rgb, refl):
            f.write("%d %d %d %d %d %d %d\n" % (p[0], p[1], p[2], c[0], c[1], c[2], r))


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [0.5, 0.3])
@pytest.mark.parametrize("transform", [0, 2])
def test_whole_codec_recolour(tmp_path, scale, transform):
    """tmc3 with the recolouring drop-in (PCCB200_DROPIN_STRICT=1: no fallback)
    against the unmodified tmc3, lossy geometry with merged duplicates, colour
    and reflectance, the input cut into several slices: bitstream, encoder
    reconstruction and decoder output md5-identical"""
    import codec_harness as ch

    if not (os.path.exists(ch.REF_BIN) and os.path.exists(RECOLOUR_BIN)):
        pytest.skip("oracle/_ref/tmc3_ref and tmc3_b200_recolour not built")
    xyz, rgb = cloud_shell(40000, bits=10, seed=31)
    rgb = texture(rgb, 24, 32)
    refl = (rgb[:, 0].astype(np.int64) * 3 + rgb[:, 2]) // 4
    ply = str(tmp_path / "in.ply")
    _write_ply(ply, xyz, rgb, refl)
    base = [f for f in (ch.enc_flags(34, transform) if transform == 0 else ch.lod_flags(34, transform))
            if not f.startswith(("--mergeDuplicatedPoints", "--positionQuantizationScale", "--attribute",
                                 "--convertPlyColourspace"))]
    flags = base + ["--mergeDuplicatedPoints=1", f"--positionQuantizationScale={scale}",
                    "--partitionMethod=4", "--sliceMaxPoints=15000", "--sliceMinPoints=5000",
                    "--convertPlyColourspace=0",
                    "--attribute=color", "--bitdepth=16", "--attribute=reflectance"]

    def md5(path):
        return hashlib.md5(open(path, "rb").read()).hexdigest()

    env = dict(os.environ, PCCB200_DROPIN_STRICT="1")
    out = {}
    for name, binary in (("ref", ch.REF_BIN), ("b200", RECOLOUR_BIN)):
        b, r = str(tmp_path / f"{name}.bin"), str(tmp_path / f"{name}_rec.ply")
        cmd = [binary, f"--uncompressedDataPath={ply}", f"--compressedStreamPath={b}",
               f"--reconstructedDataPath={r}"] + flags
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
        assert res.returncode == 0, res.stdout[-2000:]
        out[name] = (b, r, res.stdout)
    slices = re.search(r"Slice number: (\d+)", out["ref"][2])
    assert slices and int(slices.group(1)) > 1, "one slice only"
    assert md5(out["ref"][0]) == md5(out["b200"][0]), "bitstreams differ"
    assert md5(out["ref"][1]) == md5(out["b200"][1]), "encoder reconstructions differ"
    dec = {}
    for name, binary in (("ref", ch.REF_BIN), ("b200", RECOLOUR_BIN)):
        d = str(tmp_path / f"d{name}.ply")
        res = subprocess.run([binary, "--mode=1", f"--compressedStreamPath={out['ref'][0]}",
                              f"--reconstructedDataPath={d}", "--convertPlyColourspace=0"],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
        assert res.returncode == 0, res.stdout[-2000:]
        dec[name] = md5(d)
    assert dec["ref"] == dec["b200"]
