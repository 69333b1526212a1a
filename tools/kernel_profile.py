#!/usr/bin/env python
"""Developer tool: per-launch time of every engine kernel in the testing-mode forward, from torch.profiler (CUDA activity):

    python tools/kernel_profile.py [--n 1000] [--batch 256] [--precision fp16x3] [--forwards 3] [--label NAME]

Three warm-up forwards, then `--forwards` profiled ones.  Prints one JSON line: the label, the card, and per kernel name
{"us_per_launch", "launches"}.  Set POINTDSC_B200_LIB to profile another build of the library."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pointdsc_b200 import PointDSC  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--precision", default="fp16x3")
    ap.add_argument("--forwards", type=int, default=3)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool times the engine's kernels")
    m = PointDSC(num_layers=12, k=40, precision=args.precision, **bench.CTOR["3dmatch"])
    m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False)
    m = m.cuda().eval()
    h = bench.make_inputs(args.n, args.batch, "3dmatch", 0)
    d = [h[x].cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    for _ in range(3):
        m.run(*d)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.forwards):
            m.run(*d)
        torch.cuda.synchronize()
    out = {"label": args.label, "gpu": torch.cuda.get_device_name(0), "n": args.n, "batch": args.batch,
           "precision": args.precision, "forwards": args.forwards}
    for e in sorted(prof.key_averages(), key=lambda e: e.key):
        total = getattr(e, "device_time_total", None)
        if total is None:
            total = e.cuda_time_total
        if "pdsc::" in e.key and e.count and total:
            out[e.key] = {"us_per_launch": round(total / e.count, 1), "launches": e.count}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
