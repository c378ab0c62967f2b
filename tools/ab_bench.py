"""Developer tool (needs a GPU): old against new in one command.

    ab_bench.py OLD_TREE [runs] [steps] [warmup]

OLD_TREE is a second, built copy of the repository (for instance the parent
commit exported and built next to this one).  Runs `bench.py --gpus 1 --steps
K --warmup W --dump-outputs DIR` of the two trees alternately, `runs` times
each, one process at a time (a step's workspace is ~55 GB), prints the
figures that matter per run with the sampled clocks, and compares the dumped
.npy files of the two builds with np.array_equal.  Card name and power limit
are printed first: they are part of every number."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
old_root = os.path.abspath(sys.argv[1])
runs = int(sys.argv[2]) if len(sys.argv) > 2 else 3
steps = sys.argv[3] if len(sys.argv) > 3 else "10"
warmup = sys.argv[4] if len(sys.argv) > 4 else "3"
print("# " + subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True).stdout.strip(), flush=True)


def get(d, path):
    for k in path.split("."):
        d = d.get(k) if isinstance(d, dict) else None
    return d


KEYS = ("value", "e2e.value", "ms_per_step", "single_frame.ms", "smooth_frame.value",
        "decoder.batch.mpoints_per_s", "roofline.avg_launch_ms", "clocks.sm_mhz", "clocks.reasons",
        "parity_checked", "e2e.equals_device_resident_result", "decoder.reproduces_encoder_reconstruction",
        "decoder.batch.reproduces_encoder_reconstruction")
tmp = tempfile.mkdtemp(prefix="ab_bench_")
results = {"old": [], "new": []}
dumps = {}
for r in range(runs):
    for name, root in (("old", old_root), ("new", ROOT)):
        dump = os.path.join(tmp, f"{name}{r}")
        out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", steps,
                              "--warmup", warmup, "--dump-outputs", dump], cwd=root, capture_output=True,
                             text=True)
        lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
        if out.returncode != 0 or not lines:
            print(out.stderr[-2000:])
            raise SystemExit(f"{name} run {r}: bench.py failed ({out.returncode})")
        res = json.loads(lines[-1])
        results[name].append(res)
        dumps.setdefault(name, dump)
        print(f"{name} run {r}: " + ", ".join(f"{k} {get(res, k)}" for k in KEYS), flush=True)

same = True
for f in sorted(os.listdir(dumps["old"])):
    a, b = np.load(os.path.join(dumps["old"], f)), np.load(os.path.join(dumps["new"], f))
    eq = bool(np.array_equal(a, b))
    same &= eq
    print(f"dump {f}: {'identical' if eq else 'DIFFERENT'} {a.shape}")
for k in ("value", "e2e.value", "single_frame.ms", "smooth_frame.value", "decoder.batch.mpoints_per_s"):
    o = sorted(get(x, k) for x in results["old"])
    nw = sorted(get(x, k) for x in results["new"])
    print(f"{k}: old min/median/max {o[0]:.2f} {o[len(o) // 2]:.2f} {o[-1]:.2f} | "
          f"new {nw[0]:.2f} {nw[len(nw) // 2]:.2f} {nw[-1]:.2f} | median ratio {nw[len(nw) // 2] / o[len(o) // 2]:.3f}")
print("all dumps identical:", same)
sys.exit(0 if same else 1)
