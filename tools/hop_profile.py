"""Developer tool (needs a GPU): where the cycles of a block of the RDOQ
encoder descent go, one frame alone and one step of the bench workload, from
the cycle counters of the developer build

    make -C mpeg-pcc-tmc13_b200 hopstats
    hop_profile.py [frames per step] [distinct frames]

together with the per-phase times of the same calls (profile_read), the card's
name and its power limit.  Counters are sums over all units by lane 0 of each
warp; the PCCB200_* tuning numbers in the environment apply."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mpeg-pcc-tmc13_b200"))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import numpy as np  # noqa: E402
import torch  # noqa: E402
import pcc_attr_b200 as pb  # noqa: E402
import bench  # noqa: E402

COUNTERS = ("blocks", "child_polls", "child_cycles", "classify_cycles", "tz_calls",
            "tz_polls", "tz_cycles", "tail_cycles", "extra_loads", "walk1", "walk2", "walk3_4",
            "walk5_8", "walk9_")
STEPS = 32

pb.LIB_PATH = os.path.join(ROOT, "mpeg-pcc-tmc13_b200", "build", "hopstats", "libpcc_attr_b200.so")
lib = pb.lib()
if not hasattr(lib, "pccb200_hop_stats_read"):
    raise SystemExit("hop_profile.py needs the developer build: make -C mpeg-pcc-tmc13_b200 hopstats")

F = int(sys.argv[1]) if len(sys.argv) > 1 else bench.FRAMES_PER_STEP
D = int(sys.argv[2]) if len(sys.argv) > 2 else 8
print("# " + subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True).stdout.strip())
print("# env: " + " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("PCCB200_")))
dev = torch.device("cuda", 0)
pb.set_device(0)
p, q = bench.make_pods(pb)
src = []
for i in range(D):
    xyz, rgb, refl = bench.make_frame(2 + i)
    src.append((torch.from_numpy(xyz).to(dev), torch.from_numpy(rgb).to(dev), torch.from_numpy(refl).to(dev)))
n = src[0][0].shape[0]
units = []
for u in range(F):
    x, r, l = src[u % D]
    units.append({"xyz": x, "rgb0": r, "refl0": l, "rgb": torch.empty_like(r), "refl": torch.empty_like(l),
                  "crgb": torch.empty((3, n), dtype=torch.int32, device=dev),
                  "crefl": torch.empty((1, n), dtype=torch.int32, device=dev)})


def step(sub):
    for d in sub:
        d["rgb"].copy_(d["rgb0"])
        d["refl"].copy_(d["refl0"])
    torch.cuda.synchronize()
    pb.time_begin()
    pb.attr_raht_multi_batch_dev(True, p, [q, q], [d["xyz"].data_ptr() for d in sub],
                                 [[d["rgb"].data_ptr(), d["refl"].data_ptr()] for d in sub],
                                 [[d["crgb"].data_ptr(), d["crefl"].data_ptr()] for d in sub],
                                 [n] * len(sub), [3, 1])
    return pb.time_end()


def read_stats():
    buf = (C.c_uint64 * (STEPS * len(COUNTERS)))()
    got = lib.pccb200_hop_stats_read(buf, C.c_int32(STEPS))
    if got != len(COUNTERS):
        raise SystemExit(f"pccb200_hop_stats_read: {got} counters per step, expected {len(COUNTERS)}")
    return np.array(buf[:], dtype=np.float64).reshape(STEPS, len(COUNTERS))


def report(label, sub):
    step(sub)
    read_stats()
    ms = step(sub)
    st = read_stats()
    pb.profile_reset()
    pb.profile_enable(True)   # (events around every launch: its own run, not the timed one)
    step(sub)
    pb.profile_enable(False)
    read_stats()
    pr = pb.profile_read()
    print(f"\n== {label}: {len(sub)} frame(s) of {n} points, {ms:.1f} ms "
          f"({len(sub) * n / ms / 1e3:.1f} Mpoints/s)")
    print("   phase_ms (sum over launches, all lanes): "
          + ", ".join(f"{k} {v[0]:.1f} ({v[1]})" for k, v in pr.items() if v[1]))
    tot = st.sum(axis=0)
    c = dict(zip(COUNTERS, tot))
    b = max(c["blocks"], 1.0)
    walks = max(c["tz_calls"], 1.0)
    print(f"   blocks {int(c['blocks'])}; per block, cycles: child poll {c['child_cycles'] / b:.0f}, "
          f"values in -> state word {c['classify_cycles'] / b:.0f}, look-backs {c['tz_cycles'] / b:.0f}, "
          f"last look-back -> st_rec {c['tail_cycles'] / b:.0f}")
    print(f"   per block, sleeps: child poll {c['child_polls'] / b:.2f}, "
          f"look-back {c['tz_polls'] / b:.2f}; look-backs {c['tz_calls'] / b:.2f}, "
          f"loads beyond the prefetched words {c['extra_loads'] / b:.2f}")
    print("   words read per look-back: "
          + ", ".join(f"{nm[4:]}: {100 * c[nm] / walks:.1f} %" for nm in COUNTERS[9:]))
    print("   per descent step: blocks | child poll, classify, look-back, tail cycles per block | sleeps per block")
    for d in range(STEPS):
        if st[d, 0] > 0:
            r = dict(zip(COUNTERS, st[d]))
            bb = r["blocks"]
            print(f"   step {d:2d}: {int(bb):9d} | {r['child_cycles'] / bb:8.0f} {r['classify_cycles'] / bb:6.0f} "
                  f"{r['tz_cycles'] / bb:8.0f} {r['tail_cycles'] / bb:6.0f} | "
                  f"child {r['child_polls'] / bb:7.2f} look-back {r['tz_polls'] / bb:7.2f}")


report("one frame alone", units[:1])
report("one step", units)
