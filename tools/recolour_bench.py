"""Developer tool (needs a GPU): recolouring colour and reflectance of the
bench.py frame, one set per call against all sets per call, and many frames
per call.

    recolour_bench.py [frames] [repeats]

Geometry: bench.py's 1M-point synthetic LiDAR frames (RGB + 8-bit
reflectance), recoloured onto the half-resolution, duplicate-merged geometry of
bench.py's recolouring block (scale 0.5, defaults of tmc3/TMC3.cpp:1500-1551).
Timed, each after a warm-up call, median of `repeats`:

  (a) two pccb200_recolour calls (colour, then reflectance), frame 0
  (b) one pccb200_recolour_multi call (both sets), frame 0
  (c) one pccb200_recolour_multi_batch call over `frames` frames (default 16)
  (d) pccb200_recolour_multi_batch_dev over the same frames, inputs resident on
      the device (torch CUDA tensors)

  (e) one pccb200_recolour_exact_multi_batch call (both sets), frame 0: the
      reference-exact path (nanoflann's trees and search) against (b)
  (f) pccb200_recolour_exact_multi_batch_dev over the same frames, against (d)

Every call synchronises before it returns, so each figure is host wall clock
around the call; (a) to (c) and (e) include the pageable host copies.  The
outputs of (a) to (d) are compared, and those of (e) with (f).  For (b) and
(e) one more call runs with the library's phase timer on: phase "sort" is the
grid build or the two tree builds, "block_transform" the searches, forward
colours and backward lists, "tail" the final colours; the kernel launches of
one call are counted.  The registers and stack of the tree search kernel
(ptxas, from the library's build log) and the card's name and power limit are
printed with the numbers."""
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


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    import torch

    import bench
    import pcc_attr_b200 as pb

    if not torch.cuda.is_available():
        raise SystemExit("recolour_bench.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    src, attrs, tgt = [], [], []
    for f in range(frames):
        xyz, rgb, refl = bench.make_frame(2 + f)
        src.append(xyz)
        attrs.append([rgb, refl])
        tgt.append(np.ascontiguousarray(np.unique(np.rint(xyz * 0.5).astype(np.int32), axis=0)))
    scales, offs, bds = [0.5] * frames, [(0, 0, 0)] * frames, [8, 8]
    rp = pb.default_recolour_params()
    res = {}

    def one_set_calls():
        res["a"] = [pb.recolour(rp, src[0], a, tgt[0], 0.5) for a in attrs[0]]

    def multi():
        res["b"] = pb.recolour_multi(rp, src[0], attrs[0], tgt[0], 0.5, (0, 0, 0), bds)

    def batch():
        res["c"] = pb.recolour_multi_batch(rp, src, attrs, tgt, scales, offs, bds)

    dev = torch.device("cuda")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dsrc, dtgt = [T(x) for x in src], [T(x) for x in tgt]
    dattrs = [[T(a) for a in u] for u in attrs]
    douts = [[torch.empty((t.shape[0], a.shape[1]), dtype=torch.int32, device=dev) for a in u]
             for t, u in zip(tgt, attrs)]
    torch.cuda.synchronize()

    def batch_dev():
        pb.recolour_multi_batch_dev(rp, dsrc, dattrs, dtgt, scales, offs, douts, bds)

    out = {"card": card, "source_points_per_frame": int(src[0].shape[0]),
           "target_points_frame0": int(tgt[0].shape[0]), "frames": frames, "repeats": repeats}
    for key, fn in (("a_two_recolour_calls", one_set_calls), ("b_recolour_multi", multi),
                    (f"c_multi_batch_{frames}_frames", batch), (f"d_multi_batch_dev_{frames}_frames", batch_dev)):
        med, best = timed(fn, repeats)
        out[key] = {"ms_median": med, "ms_min": best}
        if "batch" in key:
            out[key]["ms_per_frame"] = med / frames
    def exact():
        res["e"] = pb.recolour_exact_multi_batch(rp, [src[0]], [attrs[0]], [tgt[0]], [0.5], [(0, 0, 0)], bds)[0]

    eouts = [[torch.empty_like(o) for o in u] for u in douts]

    def exact_dev():
        pb.recolour_exact_multi_batch_dev(rp, dsrc, dattrs, dtgt, scales, offs, eouts, bds)

    for key, fn in (("e_exact_multi_batch_1_frame", exact), (f"f_exact_multi_batch_dev_{frames}_frames", exact_dev)):
        med, best = timed(fn, repeats)
        out[key] = {"ms_median": med, "ms_min": best}
        if "dev" in key:
            out[key]["ms_per_frame"] = med / frames

    # per-phase device time and launches of one call, grid (b) and exact (e)
    for key, fn in (("phases_b_grid", multi), ("phases_e_exact", exact)):
        pb.profile_reset()
        pb.profile_enable(True)
        before = pb.kernel_launch_count()
        fn()
        launches = pb.kernel_launch_count() - before
        pb.profile_enable(False)
        prof = pb.profile_read()
        out[key] = {"launches": int(launches),
                    "ms": {n: round(v[0], 3) for n, v in prof.items() if v[1]}}
    log = os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "build.log")
    if os.path.exists(log):
        lines = open(log).read().splitlines()
        for i, l in enumerate(lines):
            if "k_foreachINS_12KdKnnQueryFn" in l and "Compiling entry" in l:
                out["ptxas_KdKnnQueryFn"] = " | ".join(x.strip() for x in lines[i + 1:i + 3])
    dres = [[o.cpu().numpy() for o in u] for u in douts]
    eres = [[o.cpu().numpy() for o in u] for u in eouts]
    out["exact_batch_equals_exact_call"] = all(np.array_equal(x, y) for x, y in zip(res["e"], eres[0]))
    out["exact_differs_from_grid_targets"] = int(sum((x != y).any(axis=1).sum() for x, y in zip(res["e"], res["b"])))
    same = (all(np.array_equal(x, y) for x, y in zip(res["a"], res["b"]))
            and all(np.array_equal(x, y) for x, y in zip(res["a"], res["c"][0]))
            and all(np.array_equal(x, y) for u, v in zip(res["c"], dres) for x, y in zip(u, v)))
    out["outputs_identical"] = bool(same)
    print(json.dumps(out, indent=1))
    sys.exit(0 if same and out["exact_batch_equals_exact_call"] else 1)


if __name__ == "__main__":
    main()
