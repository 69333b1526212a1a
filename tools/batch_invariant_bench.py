#!/usr/bin/env python
"""Cost of the batch-invariant mode (PointDSC(batch_invariant=True), pdsc_set_batch_invariant) against the default mode.

    python tools/batch_invariant_bench.py [--repeats 5] [--precision fp16x3] [--out profiles/batch_invariant_bench.jsonl] [--append]

The mode's key split uses chunks of PDSC_ATTN_INVARIANT_TILES key tiles (csrc/sets.cuh, a compile-time constant).  To measure
another value, build it beside the product library and point the run at it:
    python tools/build_variant.py tsi4 -DPDSC_ATTN_INVARIANT_TILES=4
    POINTDSC_B200_LIB=$PWD/tools/bin/lib_tsi4.so python tools/batch_invariant_bench.py --append
The value a library was built with is read back from its workspace size (one partial-result slot per split work item).

Cases (seeded synthetic sets, released 3DMatch weights):
  b256_n1000    the default configuration of bench.py: one uniform call of 256 sets of N = 1000 (eager)
  bs1_n1000     the evaluation loops' bs = 1 at N = 1000: 32 calls of model.run (graph replay), time per call
  bs1_n5000     the same at N = 5000: 16 calls
  mix_3dmatch   one forward_many call over 64 sets of the 3DMatch-like mix of tools/mixed_batch_bench.py
Default and invariant mode run on two modules with the same weights, alternated within every repeat; medians are reported.
One JSON line per case, with the card's name, power limit and maximum SM clock read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

PARTIAL_BYTES = 65536 + 1024      # one split work item's partial O and (m, l) (encoder_tc.cu)
DEFAULT_PARTIAL_ITEMS = 320       # the default mode's fixed partial slots (kAttnSplitMaxItems)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    fields = (q.stdout.strip().splitlines() or ["unknown, unknown, unknown"])[0].split(", ")
    return dict(zip(("gpu", "power_limit", "sm_clock_max"), fields))


def invariant_tiles(m_def, m_inv):
    """Key tiles per split of the loaded library's invariant mode, from the workspace of one set of N = 16384 (KT = 256)."""
    lib = m_def._ensure_engine()
    m_inv._ensure_engine()
    diff = int(lib.pdsc_workspace_bytes(m_inv._engine, 1, 16384)) - int(lib.pdsc_workspace_bytes(m_def._engine, 1, 16384))
    items = diff // PARTIAL_BYTES + DEFAULT_PARTIAL_ITEMS
    return 256 // (items // 128)


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--precision", default="fp16x3")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "batch_invariant_bench.jsonl"))
    ap.add_argument("--append", action="store_true", help="append to --out instead of replacing it")
    args = ap.parse_args(argv)
    if args.repeats < 3:
        sys.exit("--repeats must be >= 3")
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    import bench
    from mixed_batch_bench import draw_sizes
    from pointdsc_b200 import PointDSC
    from pointdsc_b200.synth import make_pair

    models = {}
    for mode in ("default", "invariant"):
        m = PointDSC(num_layers=12, k=40, precision=args.precision, batch_invariant=mode == "invariant", **bench.CTOR["3dmatch"])
        m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False)
        models[mode] = m.cuda().eval()
    tsi = invariant_tiles(models["default"], models["invariant"])
    info = card()

    def device(h):
        return [h[k].cuda() for k in ("corr_pos", "src_keypts", "tgt_keypts")]

    big = device(bench.make_inputs(1000, 256, "3dmatch", 0))
    one_1k = device(bench.make_inputs(1000, 1, "3dmatch", 0))
    one_5k = device(bench.make_inputs(5000, 1, "3dmatch", 0))
    sizes = draw_sizes("3dmatch", 64, 101)
    mix = []
    for i, n in enumerate(sizes):
        p = make_pair(10_000 + i, n, "3dmatch", 0.3)
        mix.append({k: p[k].cuda()[None] for k in ("corr_pos", "src_keypts", "tgt_keypts")})
        mix[-1]["testing"] = True

    cases = {
        "b256_n1000": (1, lambda m: m.run(*big)),
        "bs1_n1000": (32, lambda m: [m.run(*one_1k) for _ in range(32)]),
        "bs1_n5000": (16, lambda m: [m.run(*one_5k) for _ in range(16)]),
        "mix_3dmatch": (1, lambda m: m.forward_many(mix)),
    }
    lines = []
    for name, (calls, fn) in cases.items():
        for m in models.values():       # warm-up: modules, graphs, workspaces
            fn(m)
            fn(m)
        times = {mode: [] for mode in models}
        for _ in range(args.repeats):
            for mode, m in models.items():
                times[mode].append(timed(lambda: fn(m)) / calls)
        med = {mode: statistics.median(v) for mode, v in times.items()}
        rec = {"tool": "batch_invariant_bench", "case": name, "tsi": tsi, "precision": args.precision, "repeats": args.repeats,
               "seconds_per_call_median": med, "seconds_per_call_all": times,
               "invariant_over_default": med["invariant"] / med["default"], **info}
        if name == "mix_3dmatch":
            rec.update(sets=len(sizes), rows=sum(sizes), n_min=min(sizes), n_max=max(sizes))
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a" if args.append else "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
