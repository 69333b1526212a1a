#!/usr/bin/env python
"""Throughput of evaluate.py's loop (matching, labels, forward, statistics) with and without packed groups.

    python tools/packed_eval_bench.py [--pairs 64] [--repeats 5] [--group 8] [--out profiles/packed_eval_bench.jsonl]

Seeded synthetic descriptor pairs: unit FCGF-like descriptors (D = 32, float32) with planted matches (40 % of the sources are
noisy copies of a target descriptor, their key points mapped by the pair's ground-truth transform), N drawn from
tools/mixed_batch_bench.py's 3DMatch-like mix, the target count within 10 % of it.  Key points and descriptors are held in host
memory and copied to the device as the data-set path of evaluate.py loads them (evaluate.to_device), one pair at a time
inside the loop.
Arms, alternated within every repeat, each with and without the mutual check, medians of pairs/s reported:
  bs1          evaluate(batch_size=1): match, labels, forward and statistics per pair
  per_pair_P   the group loop before packed groups, restated here: per pair `match` (which then ended in a read of the
               correspondence count) and a pageable upload of gt_trans, then one `forward_many` per group and `eval_stats` per pair
  packed_P     evaluate(batch_size=P): one match_many, forward_packed and eval_stats_packed per group
One JSON line per mutual setting, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def make_pairs(count, seed, D=32):
    """[(scene index, (src xyz, src desc), (tgt xyz, tgt desc), gt_trans)] as host arrays."""
    from mixed_batch_bench import draw_sizes
    from pointdsc_b200.synth_scene import rigid
    unit = lambda f: f / np.linalg.norm(f, axis=1, keepdims=True)      # noqa: E731
    rng = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(draw_sizes("3dmatch", count, seed)):
        nt = int(n * rng.uniform(0.9, 1.1))
        R, t = rigid(1000 + i)
        tk = rng.uniform(-2, 2, (nt, 3))
        td = unit(rng.standard_normal((nt, D)))
        sk = rng.uniform(-2, 2, (n, 3))
        sd = unit(rng.standard_normal((n, D)))
        k = int(0.4 * n)
        idx = rng.integers(0, nt, k)
        sd[:k] = unit(td[idx] + 0.1 / np.sqrt(D) * rng.standard_normal((k, D)))
        sk[:k] = (tk[idx] - t) @ R + 0.01 * rng.standard_normal((k, 3))           # R sk + t = tk, up to noise
        gt = np.eye(4)
        gt[:3, :3], gt[:3, 3] = R, t
        out.append((i % 2, (sk.astype(np.float32), sd.astype(np.float32)), (tk.astype(np.float32), td.astype(np.float32)), gt))
    return out


def loaded(host_pairs, device):
    """The pairs as the loop sees them: each copied to the device when the loop asks for it."""
    import evaluate
    for si, (sx, sd), (tx, td), gt in host_pairs:
        yield (si, (evaluate.to_device(sx, device), evaluate.to_device(sd, device)),
               (evaluate.to_device(tx, device), evaluate.to_device(td, device)), gt)


@torch.no_grad()
def per_pair_groups(model, pairs, cfg, use_mutual, batch_size, device="cuda"):
    """The group loop of evaluate.py before packed groups: pairs matched one by one, every `batch_size` of them through one
    forward_many, then eval_stats pair by pair; the statistics read once at the end."""
    import evaluate
    from pointdsc_b200.frontend import match
    from pointdsc_b200.metrics import eval_stats
    rows, group = [], []

    def run_group():
        for (data, gt_t, labels), res in zip(group, model.forward_many([g[0] for g in group])):
            rows.append(eval_stats(res["final_trans"], gt_t[None], data["src_keypts"], data["tgt_keypts"], res["final_labels"],
                                   labels, re_thre=cfg["re_thre"], te_thre=cfg["te_thre"]))
        group.clear()

    for si, (src_xyz, src_desc), (tgt_xyz, tgt_desc), gt in pairs:
        data = match(src_desc, tgt_desc, src_xyz, tgt_xyz, use_mutual=use_mutual)
        torch.cuda.current_stream().synchronize()          # match ended in a read of the correspondence count
        gt_t = torch.from_numpy(np.asarray(gt, dtype=np.float32)).to(device)
        labels = evaluate.gt_labels(data, gt_t, cfg["inlier_threshold"])
        data["testing"] = True
        group.append((data, gt_t, labels))
        if len(group) == batch_size:
            run_group()
    if group:
        run_group()
    return torch.cat(rows, 0).double().cpu().numpy()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--group", type=int, default=8)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "packed_eval_bench.jsonl"))
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this benchmark measures the GPU")
    import evaluate
    from mixed_batch_bench import card
    cfg = evaluate.load_config("PointDSC_3DMatch_release")
    model = evaluate.build_model("PointDSC_3DMatch_release", cfg, "cuda")
    host = make_pairs(args.pairs, 7)
    name, power = card()
    P = args.group
    lines = []
    for mutual in (False, True):
        arms = {"bs1": lambda: evaluate.evaluate(model, loaded(host, "cuda"), cfg, use_mutual=mutual, batch_size=1),
                f"per_pair_{P}": lambda: per_pair_groups(model, loaded(host, "cuda"), cfg, mutual, P),
                f"packed_{P}": lambda: evaluate.evaluate(model, loaded(host, "cuda"), cfg, use_mutual=mutual, batch_size=P)}
        results = {}
        for k, fn in arms.items():           # warm-up: modules, graphs, workspaces, page-locked staging
            results[k] = fn()
        times = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()                         # every arm ends in its one read of the statistics
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
        med = {k: statistics.median(v) for k, v in times.items()}
        sizes = [len(p[1][0]) for p in host]
        rec = {"tool": "packed_eval_bench", "mutual": mutual, "pairs": len(host), "group": P, "n_min": min(sizes),
               "n_max": max(sizes), "n_mean": float(np.mean(sizes)), "descriptor": "fp32 D=32", "precision": model.precision,
               "repeats": args.repeats, "pairs_per_s": {k: len(host) / v for k, v in med.items()}, "seconds_median": med,
               "seconds_all": times, "success": {k: float(r[:, 0].mean()) for k, r in results.items()}, "gpu": name,
               "power_limit": power}
        rec["packed_over_per_pair"] = med[f"per_pair_{P}"] / med[f"packed_{P}"]
        rec["packed_over_bs1"] = med["bs1"] / med[f"packed_{P}"]
        print(json.dumps(rec))
        lines.append(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
