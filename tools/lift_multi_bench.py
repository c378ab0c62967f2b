"""Developer tool (needs a GPU): lifting colour and reflectance of the bench.py
frame, one attribute per call against all attributes per call, and many frames
per call.

    lift_multi_bench.py [frames] [repeats]

Input: bench.py's 1M-point synthetic LiDAR frames (RGB + 8-bit reflectance).
LoD parameters as bench_workloads.py's lifting workload (distance decimation,
sampling period 4, three neighbours), run with 12 and then with 3 levels of
detail; colour with last-component prediction.  Timed, each after a warm-up
call, median of `repeats`:

  (a) two pccb200_attr_lift_encode calls (colour, then reflectance), frame 0
  (b) a pccb200_lod_handle and two pccb200_attr_lift_encode_lod calls, frame 0
      (handle creation included)
  (c) one pccb200_attr_lift_encode_multi call (both sets), frame 0
  (d) one pccb200_attr_lift_encode_multi_batch call over `frames` frames
      (default 16)
  (e) pccb200_attr_lift_encode_multi_batch_dev over the same frames, inputs
      resident on the device (torch CUDA tensors)

Every call synchronises before it returns, so each figure is host wall clock
around the call; (a) to (d) include the pageable host copies.  The outputs of
(a) to (e) are compared; the card's name and power limit are printed with the
numbers."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), 1e3 * min(ts)


def lod_params(pb, levels):
    lp = pb.LodParams()
    lp.num_detail_levels, lp.lod_decimation_type, lp.dist2 = levels, 0, 0
    lp.num_pred_nearest_neighbours, lp.inter_lod_search_range = 3, 1100000
    lp.intra_lod_search_range, lp.intra_lod_prediction_skip_layers = 0, 0x7fffffff
    lp.prediction_with_distribution = 1
    for i in range(3):
        lp.lod_neigh_bias[i] = 1
    for i in range(32):
        lp.lod_sampling_period[i] = 4
    return lp


def qpset(pb, qp, chroma):
    q = pb.QpSet()
    q.num_layers, q.max_qp, q.fixed_point_qp_offset = 1, 51, 24
    q.layers[0][0], q.layers[0][1] = qp, chroma
    return q


def run_levels(pb, torch, levels, frames, repeats):
    import bench

    lp = lod_params(pb, levels)
    qs = [qpset(pb, bench.QP, bench.CHROMA_OFFSET), qpset(pb, bench.QP, 0)]
    en, bd = [1, 0], [8, 8]
    xyzs, attrs = [], []
    for f in range(frames):
        xyz, rgb, refl = bench.make_frame(2 + f)
        xyzs.append(np.ascontiguousarray(xyz, dtype=np.int32))
        attrs.append([np.ascontiguousarray(rgb, dtype=np.int32), np.ascontiguousarray(refl, dtype=np.int32)])
    lib = pb.lib()
    res = {}

    def one_set_calls():
        res["a"] = [pb.attr_lift_encode(lp, qs[s], xyzs[0], attrs[0][s], en[s], bd[s]) for s in range(2)]

    def handle_calls():
        h = C.c_void_p()
        pb._check(lib.pccb200_lod_create(C.byref(lp), pb._p(xyzs[0], C.c_int32), C.c_int32(xyzs[0].shape[0]),
                                         C.byref(h)))
        try:
            out = []
            for s in range(2):
                rec = attrs[0][s].copy()
                vals = np.zeros_like(rec)
                lcp = np.zeros(pb.MAX_LODS, dtype=np.int8)
                pb._check(lib.pccb200_attr_lift_encode_lod(
                    h, C.byref(qs[s]), C.c_int32(en[s]), None, pb._p(rec, C.c_int32), C.c_int32(rec.shape[1]),
                    C.c_int32(bd[s]), pb._p(vals, C.c_int32), pb._p(lcp, C.c_int8)))
                out.append((vals, rec, lcp[:levels].copy()))
            res["b"] = out
        finally:
            lib.pccb200_lod_destroy(h)

    def multi():
        v, r, l = pb.attr_lift_multi_encode(lp, qs, xyzs[0], attrs[0], en, bd)
        res["c"] = list(zip(v, r, l))

    def batch():
        v, r, l = pb.attr_lift_multi_batch(True, [lp] * frames, qs, xyzs, attrs, en, bd)
        res["d"] = [list(zip(*u)) for u in zip(v, r, l)]

    dev = torch.device("cuda")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dxyz = [T(x) for x in xyzs]
    dsrc = [[T(a) for a in u] for u in attrs]
    dattrs = [[torch.empty_like(a) for a in u] for u in dsrc]
    dvals = [[torch.empty_like(a) for a in u] for u in dsrc]
    rows = np.zeros((frames, 2, pb.MAX_LODS), dtype=np.int8)
    torch.cuda.synchronize()

    def batch_dev():
        for u, v in zip(dattrs, dsrc):  # (the call codes the attributes in place)
            for a, b in zip(u, v):
                a.copy_(b)
        torch.cuda.synchronize()
        pb.attr_lift_multi_batch_dev(True, [lp] * frames, qs, dxyz, dattrs, dvals, rows, en, bd)

    out = {"levels": levels}
    for key, fn in (("a_two_attr_lift_encode_calls", one_set_calls), ("b_handle_two_lod_calls", handle_calls),
                    ("c_attr_lift_encode_multi", multi), (f"d_multi_batch_{frames}_frames", batch),
                    (f"e_multi_batch_dev_{frames}_frames", batch_dev)):
        med, best = timed(fn, repeats)
        out[key] = {"ms_median": med, "ms_min": best}
        if "batch" in key:
            out[key]["ms_per_frame"] = med / frames
    same = lambda x, y: all(np.array_equal(p, q) for p, q in zip(x, y))
    ok = all(same(res["a"][s], res[k][s]) for k in ("b", "c") for s in range(2))
    ok = ok and all(same(res["a"][s], res["d"][0][s]) for s in range(2))
    for f in range(frames):
        for s in range(2):
            dv = (dvals[f][s].cpu().numpy(), dattrs[f][s].cpu().numpy(), rows[f, s, :levels])
            ok = ok and same(res["d"][f][s], dv)
    out["outputs_identical"] = bool(ok)
    return out


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    import torch

    import pcc_attr_b200 as pb

    if not torch.cuda.is_available():
        raise SystemExit("lift_multi_bench.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = {"card": card, "frames": frames, "repeats": repeats,
           "runs": [run_levels(pb, torch, levels, frames, repeats) for levels in (12, 3)]}
    print(json.dumps(out, indent=1))
    sys.exit(0 if all(r["outputs_identical"] for r in out["runs"]) else 1)


if __name__ == "__main__":
    main()
