"""Times the predicting-transform decoder (pccb200_attr_pred_decode_multi_batch)
on the GPU: one unit, and many units per call, for a 12-level slice with
intra-LoD prediction (the CTC near-lossless form) and a single-level slice.
The baseline is the plain-C restatement of the reference's decode loop
(oracle/pred_oracle.c) on one core, which also checks every output.  Reports
the dependency depth of each slice's predictor DAG (the longest chain of
neighbour references), which bounds the dataflow's critical path.

    python tools/pred_decode_bench.py [--n 1000000] [--units 16] [--reps 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "mpeg-pcc-tmc13_b200")]

import pcc_attr_b200 as pb  # noqa: E402
from pred_cases import make_case, oracle_pred_decode  # noqa: E402


def dag_depth(preds):
    """1 + the longest chain of neighbour references ending at each predictor"""
    n = len(preds)
    cnt = preds["neighbor_count"].tolist()
    nb = preds["predictor_index"].tolist()
    depth = [0] * n
    for i in range(n):
        d = 0
        for j in range(cnt[i]):
            x = depth[nb[i][j]]
            d = x if x > d else d
        depth[i] = d + 1
    return max(depth) if n else 0


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--units", type=int, default=16)
    ap.add_argument("--unit-n", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    gpu = torch.cuda.get_device_name(0)
    res = {"gpu": gpu}
    for name, kw in (("12_levels_intra", dict(levels=12, skip=0, blending=1, icp=1)),
                     ("single_level", dict(levels=1, skip=0, avg_disabled=1, icp=1))):
        c = make_case(n=args.n, a=3, seed=2, **kw)
        exp = oracle_pred_decode(c)
        t_cpu = timed(lambda: oracle_pred_decode(c), 1)
        batch = dict(lods=[c["lod"]], quant_neigh_weights=[c["qnw"]], qpsets=[c["qs"]],
                     preds=[c["pp"]], xyzs=[c["xyz"]], values=[[c["values"]]], bitdepths=[8],
                     icps=[[c["icp"]]])
        out = pb.attr_pred_decode_multi_batch(**batch)
        assert np.array_equal(out[0][0], exp)
        h = pb.lod_import(c["preds"], c["idx"], c["npl"], c["levels"])
        t_lod = timed(lambda: pb.attr_pred_decode_lod(h, c["qs"], c["pp"], c["qnw"], c["values"],
                                                      icp=c["icp"]), args.reps)
        pb.lod_destroy(h)
        t_one = timed(lambda: pb.attr_pred_decode_multi_batch(**batch), args.reps)
        us = [make_case(n=args.unit_n, a=3, seed=100 + u, **kw) for u in range(args.units)]
        many = dict(lods=[u["lod"] for u in us], quant_neigh_weights=[u["qnw"] for u in us],
                    qpsets=[c["qs"]], preds=[c["pp"]], xyzs=[u["xyz"] for u in us],
                    values=[[u["values"]] for u in us], bitdepths=[8], icps=[[u["icp"]] for u in us])
        outs = pb.attr_pred_decode_multi_batch(**many)
        for u, o in zip(us, outs):
            u["qs"], u["pp"] = c["qs"], c["pp"]
            assert np.array_equal(o[0], oracle_pred_decode(u))
        t_many = timed(lambda: pb.attr_pred_decode_multi_batch(**many), args.reps)
        t_many_cpu = sum(timed(lambda u=u: oracle_pred_decode(u), 1) for u in us[:4]) * len(us) / 4
        res[name] = {
            "n": args.n, "dag_depth": dag_depth(c["preds"]),
            "cpu_loop_1core_s": round(t_cpu, 4),
            "gpu_lod_entry_s": round(t_lod, 4),
            "gpu_batch_1unit_with_lod_build_s": round(t_one, 4),
            "units": args.units, "unit_n": args.unit_n,
            "unit_dag_depth": dag_depth(us[0]["preds"]),
            "gpu_batch_units_s": round(t_many, 4),
            "cpu_loop_units_1core_s": round(t_many_cpu, 4),
        }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
