#!/usr/bin/env python
"""FCGF on the device (pdsc_fcgf_packed): one group call against one call per cloud, the time split between quantisation with
the neighbour tables, each convolution and the head, and each convolution's achieved FLOP/s and gathered bytes/s.

    python tools/fcgf_bench.py [--out profiles/fcgf_bench.jsonl] [--repeats 5]

Configurations: 16 synth_scene clouds of 60,000 points at voxel 0.05 with conv1 kernel 7 (3DMatch weights), and 8 clouds of
120,000 points spread over a 60 m scene at voxel 0.30 with kernel 5 (KITTI-like).  Weights are seeded random (the released ones
are not shipped); the arithmetic does not depend on their values.  A convolution's FLOPs are 2 Cin Cout per neighbour-table hit
(absent neighbours are skipped a tile at a time, so this is the useful work); its gathered bytes are 4 Cin per hit.  Against the
H100 SXM data-sheet figures of 67 TFLOP/s FP32 and 3.35 TB/s; the card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def clouds_for(name):
    from pointdsc_b200.synth_scene import scene
    if name == "3dmatch_k7":
        return [scene(60000, seed=s) for s in range(16)], 0.05, 7
    return [(scene(120000, seed=s, layout_seed=11) * np.float32(20.0)) for s in range(8)], 0.30, 5


def timed(fn, repeats):
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "fcgf_bench.jsonl"))
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    from test_gpu_fcgf import model, run
    from oracle import fcgf_oracle as O
    from pointdsc_b200.fcgf import packed_call
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    gpu = card()
    lines = []
    for cfg in ("3dmatch_k7", "kitti_k5"):
        clouds, voxel, k1 = clouds_for(cfg)
        m = model(k1)
        dev = [torch.from_numpy(c).cuda() for c in clouds]
        in_off = [0]
        for c in clouds:
            in_off.append(in_off[-1] + len(c))
        pts = torch.cat(dev).contiguous()
        group = lambda: packed_call(m, pts, in_off, voxel)                                  # noqa: E731
        singles = lambda: [packed_call(m, c, [0, len(c)], voxel) for c in dev]              # noqa: E731
        group(); singles()
        t_group, t_single = timed(group, a.repeats), timed(singles, a.repeats)
        # where the group call's time goes: kernel times from one profiled call
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            group()
            torch.cuda.synchronize()
        kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                   and "memset" not in e.name.lower()]
        kernels.sort(key=lambda e: e.time_range.start)
        conv = [e for e in kernels if "fconv" in e.name]
        quant = sum(e.device_time for e in kernels if "fq_" in e.name or "hash_plan" in e.name) / 1e3
        maps = sum(e.device_time for e in kernels if "fmap" in e.name) / 1e3
        head = sum(e.device_time for e in kernels if "fhead" in e.name) / 1e3
        _, _, meta, reg, _ = run(m, clouds, cpu=False, voxel=voxel)
        layers = []
        for step, ev in zip(O.STEPS, conv):
            name, kind, level = step[0], step[1], step[2]
            table = "c1" if kind == "c1" else f"{kind}{level}"
            rows = int(reg[f"off{level}"][-1])
            hits = int((reg[table][:rows] >= 0).sum())
            cin = 1 if step[3] is None else O.FEAT_WIDTH[step[3][0]] - step[3][1]
            ms = ev.device_time / 1e3
            flops = 2.0 * hits * cin * step[6]
            gathered = 4.0 * hits * cin
            layers.append({"layer": name, "rows": rows, "hits": hits, "cin": cin, "cout": step[6], "ms": round(ms, 4),
                           "tflops": round(flops / ms / 1e9, 2), "fp32_peak_share": round(flops / ms / 1e9 / 67.0, 3),
                           "gathered_TBps": round(gathered / ms / 1e9, 3), "hbm_share": round(gathered / ms / 1e9 / 3350.0, 3)})
        rec = {"config": cfg, "gpu": gpu, "clouds": len(clouds), "points": in_off[-1], "voxel": voxel, "conv1_kernel": k1,
               "key_points": int(meta[len(clouds)]), "group_call_ms": round(t_group * 1e3, 2),
               "single_calls_ms": round(t_single * 1e3, 2), "quantise_ms": round(quant, 3), "tables_ms": round(maps, 3),
               "convolutions_ms": round(sum(l["ms"] for l in layers), 3), "head_ms": round(head, 3),
               "level_rows": [int(reg[f"off{l}"][-1]) for l in range(4)], "layers": layers}
        print(json.dumps({k: v for k, v in rec.items() if k != "layers"}))
        for l in layers:
            print("  ", json.dumps(l))
        lines.append(json.dumps(rec))
    with open(a.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
