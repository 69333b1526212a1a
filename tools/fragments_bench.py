"""Device time of the fragment stages (row f9): one synthetic 100-frame 640 x 480 fragment, and a group of 8 such fragments in one
call per stage against 8 single calls.  Writes profiles/fragments_bench.jsonl (or --out) with the card's name and power limit read
in the same run, and the peak device memory per fragment."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pointdsc_b200.fragments import extract_vertices_packed, integrate_packed   # noqa: E402
from pointdsc_b200.synth_scene import camera_path, render_rgbd                   # noqa: E402

INTR = (525.0, 525.0, 319.5, 239.5)


def frames(n, seed):
    poses = camera_path(n, seed)
    fr = [render_rgbd(p, 640, 480, *INTR) for p in poses]
    return np.stack([f[0] for f in fr]), np.stack([f[1] for f in fr]), np.linalg.inv(poses)


def run(group):
    dep = torch.from_numpy(np.concatenate([g[0] for g in group])).cuda()
    col = torch.from_numpy(np.concatenate([g[1] for g in group])).cuda()
    ext = np.concatenate([g[2] for g in group])
    off = np.concatenate([[0], np.cumsum([len(g[0]) for g in group])]).tolist()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    vol = integrate_packed(dep, col, ext, off, INTR)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    v, c, voff = extract_vertices_packed(vol)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3, vol.unit_offsets[-1], voff[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/fragments_bench.jsonl")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    frags = [frames(100, s) for s in range(8)]
    run(frags[:1])                                     # warm-up: module load
    rows = []
    for r in range(a.repeats):
        torch.cuda.reset_peak_memory_stats()
        one = run(frags[:1])
        peak1 = torch.cuda.max_memory_allocated()
        singles = [run([f]) for f in frags]
        torch.cuda.reset_peak_memory_stats()
        grp = run(frags)
        peak8 = torch.cuda.max_memory_allocated()
        rows.append({"repeat": r, "card": card, "one_fragment": {"integrate_ms": one[0], "extract_ms": one[1], "units": one[2],
                                                                   "vertices": one[3], "peak_bytes": peak1},
                     "eight_single_calls": {"integrate_ms": sum(s[0] for s in singles), "extract_ms": sum(s[1] for s in singles)},
                     "eight_in_one_call": {"integrate_ms": grp[0], "extract_ms": grp[1], "units": grp[2], "vertices": grp[3],
                                           "peak_bytes_per_fragment": peak8 / 8}})
        print(json.dumps(rows[-1]))
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        for row in rows:
            f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
