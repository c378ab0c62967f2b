"""Dependency depth of the predicting transform's predictor DAG (host only):
the longest chain of neighbour references, which bounds the critical path of
the GPU decoder's dataflow.  Levels of detail come from the plain-C LoD build
(oracle/lod_oracle.c) with the parameters of bench.py --workload predlift3m
(12 levels, intra-LoD prediction from level 0, blended weights), on the first
1M-point slice of that workload's cloud, and with one level of detail (a
cat3-like slice) on the same points.  The analogue of
tools/subsample_dag_depth.py.

    python tools/pred_dag_depth.py [--n 3000000] [--slice-points 1000000]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "mpeg-pcc-tmc13_b200")]

import pcc_attr_b200 as pb  # noqa: E402
from bench_workloads import lod_params  # noqa: E402
from pcc_attr_b200.synth import cloud_terrain, morton_slices  # noqa: E402
from pcc_testlib import oracle_lod_build  # noqa: E402


def dag_depth(preds):
    """(max, mean) over predictors of 1 + the longest chain of references"""
    cnt = preds["neighbor_count"].tolist()
    nb = preds["predictor_index"].tolist()
    depth = [0] * len(cnt)
    for i in range(len(cnt)):
        d = 0
        for j in range(cnt[i]):
            x = depth[nb[i][j]]
            d = x if x > d else d
        depth[i] = d + 1
    return max(depth), float(np.mean(depth))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=3_000_000)
    ap.add_argument("--slice-points", type=int, default=1_000_000)
    args = ap.parse_args()
    xyz, rgb = cloud_terrain(args.n)
    xyz_s, _, offs = morton_slices(xyz, [rgb], args.slice_points)
    x0 = np.ascontiguousarray(xyz_s[offs[0]:offs[1]], dtype=np.int32)
    res = {"slice_points": int(len(x0))}
    for name, levels in (("predlift3m_12_levels", 12), ("single_level", 1)):
        preds, _, npl = oracle_lod_build(lod_params(pb, levels, True), x0)
        mx, mean = dag_depth(preds)
        res[name] = {"levels": int(len(npl)), "depth_max": mx, "depth_mean": round(mean, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
