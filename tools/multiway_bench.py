#!/usr/bin/env python
"""Cost of the multiway registration's device calls (pointdsc_b200.multiway, row f7) and of one synthetic scene end to end.

    python tools/multiway_bench.py [--repeats 5] [--fragments 8] [--out profiles/multiway_bench.jsonl]

Records, one JSON line each, with the card's name and power limit read in the same run; medians over alternated repeats:
  information   device time (CUDA events) of information_matrix_packed over every pair of a synthetic scene's fragments (key
                points at 0.05, r = 0.07): one grouped call against one call per pair
  multi_scale   device time of multi_scale_icp_packed over the scene's odometry pairs: one grouped call against one call per pair
  scene         wall time of multiway.py's run_scene on the scene (register, optimise, ICP-refine, optimise), after a warm-up run,
                split into the device part (register_scene + refine_edges, each ending in its one read) and the host
                optimisation, with the ATE it reached"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--fragments", type=int, default=8)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "multiway_bench.jsonl"))
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    import multiway as driver
    from icp_bench import alternate
    from mixed_batch_bench import card
    from evaluate import build_model, load_config
    from pointdsc_b200 import multiway as mw
    name, power = card()
    lines = []

    def emit(rec):
        rec.update({"tool": "multiway_bench", "gpu": name, "power_limit": power, "repeats": args.repeats, "fragments": args.fragments})
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    data = driver.synthetic_scene(args.fragments, 0, "cuda")
    xyz = data["xyz"]
    odo, _, pairs = driver.scene_pairs(args.fragments)
    T_all = torch.from_numpy(np.array([np.linalg.inv(data["gt"][j]) @ data["gt"][i] for i, j in pairs], np.float32)).cuda()
    so = np.cumsum([0] + [int(xyz[i].shape[0]) for i, _ in pairs]).tolist()
    to = np.cumsum([0] + [int(xyz[j].shape[0]) for _, j in pairs]).tolist()
    src = torch.cat([xyz[i] for i, _ in pairs]).contiguous()
    tgt = torch.cat([xyz[j] for _, j in pairs]).contiguous()
    d_so = torch.tensor(so, dtype=torch.int32, device="cuda")
    d_to = torch.tensor(to, dtype=torch.int32, device="cuda")
    singles = [(xyz[i], xyz[j], T_all[k:k + 1], [0, int(xyz[i].shape[0])], [0, int(xyz[j].shape[0])],
                torch.tensor([0, int(xyz[i].shape[0])], dtype=torch.int32, device="cuda"),
                torch.tensor([0, int(xyz[j].shape[0])], dtype=torch.int32, device="cuda")) for k, (i, j) in enumerate(pairs)]
    arms = {"grouped": lambda: mw.information_matrix_packed(src, tgt, T_all, so, to, d_so, d_to),
            "per_pair": lambda: [mw.information_matrix_packed(*s) for s in singles]}
    med, allt = alternate(arms, args.repeats, 3)
    emit({"what": "information", "pairs": len(pairs), "rows_src": so[-1], "rows_tgt": to[-1], "ms_median": med, "ms_all": allt})

    T_odo = torch.from_numpy(np.array([data["odometry_init"][i] for i, _ in odo], np.float32)).cuda()
    arms = {"grouped": lambda: mw.multi_scale_icp_packed(xyz, odo, T_odo),
            "per_pair": lambda: [mw.multi_scale_icp_packed(xyz, [p], T_odo[k:k + 1]) for k, p in enumerate(odo)]}
    med, allt = alternate(arms, args.repeats, 1)
    emit({"what": "multi_scale", "pairs": len(odo), "ms_median": med, "ms_all": allt})

    cfg = load_config("PointDSC_3DMatch_release")
    model = build_model("PointDSC_3DMatch_release", cfg, "cuda")
    quiet = lambda *_: None  # noqa: E731
    with tempfile.TemporaryDirectory() as tmp:
        driver.run_scene(model, data, os.path.join(tmp, "warm"), log=quiet)
        runs = []
        for r in range(args.repeats):
            t0 = time.perf_counter()
            g0 = driver.register_scene(model, data, log=quiet)
            t1 = time.perf_counter()
            g1 = driver.optimise(g0, quiet)
            t2 = time.perf_counter()
            g2 = driver.refine_edges(data, g1)
            t3 = time.perf_counter()
            g = driver.optimise(g2, quiet)
            t4 = time.perf_counter()
            runs.append({"register_s": t1 - t0, "optimise_1_s": t2 - t1, "refine_s": t3 - t2, "optimise_2_s": t4 - t3,
                         "total_s": t4 - t0, "edges": [len(g0.edges), len(g1.edges), len(g.edges)],
                         "ate_cm": mw.trajectory_ate(data["gt"], g.nodes)})
    emit({"what": "scene", "pairs": len(pairs), "median": {k: statistics.median(r[k] for r in runs) for k in runs[0] if k.endswith("_s")},
          "edges": runs[0]["edges"], "ate_cm": runs[0]["ate_cm"], "runs": runs})
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
