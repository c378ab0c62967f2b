"""Developer tool (needs a GPU): scalable lifting against the distance-LoD
lifting path on the same 1M-point slice.

    scalable_lift_bench.py [repeats]

Input: bench.py's first synthetic LiDAR frame (RGB + reflectance).  Arms, each
timed with the library's device events (pccb200_time_begin / _end, CUDA events
spanning every lane) after a warm-up call, median and minimum of `repeats`:

  lod     the level-of-detail build alone: pccb200_lod_build (distance
          decimation, 12 levels, sampling as bench_workloads.py's lifting
          workload) against pccb200_lod_build_scalable (max_neigh_range 6)
  encode  colour (with last-component prediction) + reflectance in one call:
          pccb200_attr_lift_encode_multi_batch against
          pccb200_attr_lift_encode_scalable, host pointers (the pageable copies
          are inside the timed region)

The concatenation of layers searches the neighbours of earlier levels again;
its share is reported twice: as a count (query points searched again over all
query points searched, from numPointsInLod) and as time (the neighbour-search
phase of the library's per-phase profile, every pass included, over the whole
build).  The card's name and power limit are printed with the numbers, and
one JSON line closes the output."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))

SEARCH_PHASE = 2  # lod_pipeline.cuh: ex.phase(2), the neighbour search


def device_timed(pb, fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        pb.time_begin()
        fn()
        ts.append(pb.time_end())
    return float(np.median(ts)), float(min(ts))


def lod_params(pb):
    lp = pb.LodParams()
    lp.num_detail_levels, lp.lod_decimation_type, lp.dist2 = 12, 0, 0
    lp.num_pred_nearest_neighbours, lp.inter_lod_search_range = 3, 1100000
    lp.intra_lod_search_range, lp.intra_lod_prediction_skip_layers = 0, 0x7fffffff
    lp.prediction_with_distribution = 1
    for i in range(3):
        lp.lod_neigh_bias[i] = 1
    for i in range(pb.MAX_LODS):
        lp.lod_sampling_period[i] = 4
    return lp


def qpset(pb, qp, chroma):
    q = pb.QpSet()
    q.num_layers, q.max_qp, q.fixed_point_qp_offset = 1, 51, 24
    q.layers[0][0], q.layers[0][1] = qp, chroma
    return q


def research_share(npl, n):
    """(query points searched again by the concatenation, all query points searched)"""
    sizes = [int(x) for x in np.asarray(npl)[::-1]]
    on, again, total = True, 0, 0
    for r, size in enumerate(sizes):
        refined = size - (sizes[r + 1] if r + 1 < len(sizes) else 0)
        start = n - size
        if on and refined:
            if refined <= start:
                on = False
            else:
                again += start
        total += refined
    return again, total + again


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    import bench
    import pcc_attr_b200 as pb

    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    xyz, rgb, refl = bench.make_frame(2)
    xyz = np.ascontiguousarray(xyz, dtype=np.int32)
    rgb = np.ascontiguousarray(rgb, dtype=np.int32)
    refl = np.ascontiguousarray(refl, dtype=np.int32).reshape(len(xyz), 1)
    n = xyz.shape[0]
    lp = lod_params(pb)
    scal = pb.LodScalable(6, 0, 0, 0)
    qs = [qpset(pb, bench.QP, bench.CHROMA_OFFSET), qpset(pb, bench.QP, 0)]
    print(f"GPU: {gpu_info()}; slice: {n} points; repeats {repeats}")

    res = {"points": n, "gpu": gpu_info()}
    res["lod_distance_ms"] = device_timed(pb, lambda: pb.lod_build(lp, xyz), repeats)
    res["lod_scalable_ms"] = device_timed(pb, lambda: pb.lod_build_scalable(lp, scal, xyz), repeats)
    enc_d = lambda: pb.attr_lift_multi_batch(True, [lp], qs, [xyz], [[rgb, refl]],  # noqa: E731
                                             lcp_enabled=[1, 0])
    enc_s = lambda: pb.attr_lift_scalable(True, [lp], [scal], qs, [xyz], [[rgb, refl]],  # noqa: E731
                                          lcp_enabled=[1, 0])
    res["encode_distance_ms"] = device_timed(pb, enc_d, repeats)
    res["encode_scalable_ms"] = device_timed(pb, enc_s, repeats)

    _, _, npl = pb.lod_build_scalable(lp, scal, xyz)
    again, searched = research_share(npl, n)
    res["scalable_lods"] = len(npl)
    res["research_query_share"] = again / searched
    pb.profile_enable(1)
    pb.profile_reset()
    for _ in range(repeats):
        pb.lod_build_scalable(lp, scal, xyz)
    prof = pb.profile_read()
    pb.profile_enable(0)
    phase_ms = [v[0] for v in prof.values()]
    res["search_phase_share_of_build"] = phase_ms[SEARCH_PHASE] / max(sum(phase_ms), 1e-9)

    for k in ("lod_distance_ms", "lod_scalable_ms", "encode_distance_ms", "encode_scalable_ms"):
        print(f"{k:22s} median {res[k][0]:8.2f}  min {res[k][1]:8.2f}")
    print(f"scalable levels of detail: {res['scalable_lods']}; query points searched again by "
          f"the concatenation: {again} of {searched} ({100 * res['research_query_share']:.1f}%); "
          f"neighbour-search phase (every pass): {100 * res['search_phase_share_of_build']:.1f}% "
          "of the profiled scalable build")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
