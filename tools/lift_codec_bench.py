"""Developer tool (needs a GPU and oracle/_ref built from the reference tree):
the lifting drop-in in the whole codec, and its library calls.

    lift_codec_bench.py [points] [repeats]

(1) Wall clock of tmc3 encoding and then decoding one lifting frame
    (transformType=2, cfg/octree-liftt-ctc-lossless-geom-lossy-attrs.yaml, RGB,
    10 levels of detail; default 1M points, a synthetic textured shell) with
    oracle/_ref/tmc3_ref (the unmodified reference), tmc3_b200 (RAHT and LoD
    drop-ins) and tmc3_b200_lift (plus the lifting drop-in).  Wall clock, not
    user time: user time does not count the device's work.  The three
    bitstreams and reconstructions are compared by md5.
(2) What the lifting drop-in asks of the library per attribute, on the same
    frame's levels of detail (pccb200_lod_build): pccb200_lod_import plus one
    pccb200_attr_lift_encode_lod call, for RGB with LCP and for an 8-bit
    reflectance; median of `repeats`, host wall clock and device time
    (pccb200_time_begin / _end around the pair).

The card's name and power limit are read in the same run and printed with the
numbers, one JSON line."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))

REF = os.path.join(ROOT, "oracle", "_ref")


def md5(path):
    return hashlib.md5(open(path, "rb").read()).hexdigest()


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    import codec_harness as ch
    import pcc_attr_b200 as pb
    from pcc_attr_b200.synth import cloud_shell, texture
    from pcc_testlib import make_lod_params, make_qpset

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    xyz, rgb = cloud_shell(n, bits=12, seed=5)
    rgb = np.ascontiguousarray(texture(rgb, 24, 6).astype(np.int32))
    out = {"points": int(len(xyz)), "card": card.splitlines()[0] if card else "not read"}

    with tempfile.TemporaryDirectory() as tmp:
        ply = os.path.join(tmp, "in.ply")
        ch.write_ply(ply, xyz, rgb)
        flags = ch.lod_flags(34, 2, lods=10)
        env = dict(os.environ, PCCB200_DROPIN_STRICT="1")
        digests = {}
        for name in ("tmc3_ref", "tmc3_b200", "tmc3_b200_lift"):
            binary = os.path.join(REF, name)
            b, r, d = (os.path.join(tmp, f"{name}.{x}") for x in ("bin", "rec.ply", "dec.ply"))
            t0 = time.perf_counter()
            rc = subprocess.run([binary, f"--uncompressedDataPath={ply}", f"--compressedStreamPath={b}",
                                 f"--reconstructedDataPath={r}"] + flags, stdout=subprocess.DEVNULL,
                                stderr=subprocess.STDOUT, env=env).returncode
            t1 = time.perf_counter()
            rc |= subprocess.run([binary, "--mode=1", f"--compressedStreamPath={b}",
                                  f"--reconstructedDataPath={d}", "--convertPlyColourspace=1"],
                                 stdout=subprocess.DEVNULL, stderr=subprocess.STDOUT, env=env).returncode
            t2 = time.perf_counter()
            out[name] = {"encode_s": round(t1 - t0, 3), "decode_s": round(t2 - t1, 3), "rc": rc}
            digests[name] = (md5(b), md5(r), md5(d)) if rc == 0 else None
        out["outputs_identical"] = len(set(digests.values())) == 1 and None not in digests.values()

    lp = pb.LodParams.from_buffer_copy(bytes(make_lod_params(levels=11)))
    preds, idx, npl = pb.lod_build(lp, xyz)
    refl = np.ascontiguousarray(((rgb[:, :1] * 2 + rgb[:, 1:2]) // 3).astype(np.int32))
    sets = {"rgb_lcp": (rgb, 1, make_qpset(qp=34, chroma_offset=0, fixed_point_qp_offset=24)),
            "refl8": (refl, 0, make_qpset(qp=34, chroma_offset=0, fixed_point_qp_offset=24))}
    for name, (attrs, lcp, qs) in sets.items():
        q = pb.QpSet.from_buffer_copy(bytes(qs))

        def once():
            h = pb.lod_import(preds, idx, npl, lp.num_detail_levels)
            try:
                pb.attr_lift_encode_lod(h, q, attrs, lcp_enabled=lcp)
            finally:
                pb.lod_destroy(h)

        once()
        wall, dev = [], []
        for _ in range(repeats):
            pb.time_begin()
            t0 = time.perf_counter()
            once()
            wall.append(time.perf_counter() - t0)
            dev.append(pb.time_end())
        out[f"import_encode_lod_{name}_ms"] = {"wall": round(1e3 * float(np.median(wall)), 2),
                                               "device": round(float(np.median(dev)), 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
