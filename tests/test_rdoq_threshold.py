"""The RDOQ threshold of a coefficient (rdoq_code, raht_core.cuh: a float
estimate of floor(lhs / lambda), one correcting product and a closed-form index
into the rate table) against the plain definition: the first of the 37 values
of zero_run_rate for which the reference's test (tmc3/RAHT.cpp:1617-1636)
    (Dist2 << 26) < lambda * (Rate(tz) + ((Ratecoeff + 128) >> 8))
holds, Dist2 << 26 wrapping as a 64-bit shift.  Host build, no GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE_REMOVED, CODE_HARD = 1, 2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("rdoq") / "libemu_rdoq.so")
    subprocess.check_call([
        "g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-x", "c++",
        "-I" + os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "csrc"), "-I" + os.path.join(ROOT, "include"),
        "-I" + os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "emu_rdoq.cpp"),
        "-o", out])
    return C.CDLL(out)


def rates(emu):
    """the values zero_run_rate takes, ascending, with the shortest run of each"""
    out = []
    for tz in list(range(11)) + [10 + (1 << a) for a in range(30)]:
        r = emu.emu_zero_run_rate(tz)
        if not out or r != out[-1][0]:
            out.append((r, tz))
    return out


def wrap64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def plain(table, dist2, lam, rate_coeff):
    lhs = wrap64(dist2 << 26)
    rc = (rate_coeff + 128) >> 8
    for i, (r, _) in enumerate(table):
        if lhs < lam * (r + rc):
            return CODE_REMOVED if i == 0 else 2 + i
    return CODE_HARD


def run(emu, d2, lam, rc):
    d2 = np.ascontiguousarray(d2, dtype=np.int64)
    lam = np.ascontiguousarray(lam, dtype=np.int64)
    rc = np.ascontiguousarray(rc, dtype=np.int32)
    out = np.zeros(d2.size, dtype=np.int32)
    emu.emu_rdoq_codes(d2.ctypes.data_as(C.c_void_p), lam.ctypes.data_as(C.c_void_p),
                       rc.ctypes.data_as(C.c_void_p), C.c_int(d2.size), out.ctypes.data_as(C.c_void_p))
    return out


def test_rate_table_and_codes(emu):
    table = rates(emu)
    assert [r for r, _ in table] == [1, 2, 3, 5, 7, 9, 11] + [12 + 2 * a for a in range(1, 31)]
    # code -> run-length threshold as the block kernel decodes it
    assert [tz for _, tz in table] == [0, 1, 2, 3, 5, 7, 9] + [10 + (1 << (a - 1)) for a in range(1, 31)]


@pytest.mark.parametrize("mult", [25, 35])
def test_random_inputs(emu, mult):
    table = rates(emu)
    rng = np.random.default_rng(mult)
    n = 40000
    l0 = rng.integers(1, 1 << 22, size=n)
    l0[: n // 4] = rng.integers(1, 64, size=n // 4)
    lam = l0 * l0 * mult
    # left sides spread over the whole rate range and a little beyond
    ratio = rng.uniform(0.0, 90.0, size=n)
    d2 = (lam.astype(np.float64) * ratio / (1 << 26)).astype(np.int64)
    rc = rng.integers(0, 1400, size=n)
    got = run(emu, d2, lam, rc)
    exp = [plain(table, int(a), int(b), int(c)) for a, b, c in zip(d2, lam, rc)]
    assert got.tolist() == exp


@pytest.mark.parametrize("mult", [25, 35])
def test_rate_boundaries(emu, mult):
    """left sides one either side of lambda * rate for every rate"""
    table = rates(emu)
    d2s, lams, rcs = [], [], []
    for l0 in (1, 3, 181, 4096, 46341, 1 << 20, (1 << 24) + 1):
        lam = l0 * l0 * mult
        for rate_coeff in (0, 127, 128, 406, 1218, 65535):
            rc = (rate_coeff + 128) >> 8
            for r, _ in table:
                edge = lam * (r + rc)
                for lhs in (edge - (1 << 26), edge, edge + (1 << 26)):
                    for dd in (-1, 0, 1):
                        d2 = (lhs >> 26) + dd
                        if 0 <= d2 < 1 << 37:
                            d2s.append(d2)
                            lams.append(lam)
                            rcs.append(rate_coeff)
    got = run(emu, d2s, lams, rcs)
    exp = [plain(table, a, b, c) for a, b, c in zip(d2s, lams, rcs)]
    assert got.tolist() == exp


@pytest.mark.parametrize("mult", [25, 35])
def test_left_side_near_and_past_int64(emu, mult):
    """Dist2 << 26 close to 2^63 and beyond it, where the shift wraps"""
    table = rates(emu)
    rng = np.random.default_rng(7 + mult)
    d2s, lams, rcs = [], [], []
    for l0 in (1 << 20, 1 << 24, 5 << 22, 46341 << 9):
        lam = l0 * l0 * mult
        assert lam * (72 + 256) < 1 << 63
        base = [(1 << 37) - 1, 1 << 37, (1 << 37) + 1, (1 << 38) - 1, 1 << 38, (3 << 37) + 5,
                (1 << 40) + 12345, (1 << 62) + 99, (1 << 63) - 1]
        base += [int(x) for x in rng.integers(1 << 36, 1 << 39, size=500)]
        base += [int(x) for x in rng.integers(1 << 39, (1 << 63) - 1, size=500)]
        base += [int(lam * x) >> 26 for x in rng.uniform(0.0, 90.0, size=300)]
        for d2 in base:
            d2s.append(d2)
            lams.append(lam)
            rcs.append(int(rng.integers(0, 1400)))
    got = run(emu, d2s, lams, rcs)
    exp = [plain(table, a, b, c) for a, b, c in zip(d2s, lams, rcs)]
    assert got.tolist() == exp
    assert CODE_REMOVED in exp and CODE_HARD in exp
