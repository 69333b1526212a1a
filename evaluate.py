#!/usr/bin/env python
"""The reference's evaluation driver (`evaluation/test_3DMatch.py`, `--solver SVD`) with every per-pair step on the H100 and no
host synchronisation inside the loop: descriptor matching + network input (row f1, `pointdsc_b200.frontend.match`), ground-truth
labels, `PointDSC.forward` (the path), registration + classification statistics (row f3, `pointdsc_b200.metrics.eval_stats`);
with --batch_size P every P pairs take one call of each (`match_many`, `forward_packed`, `eval_stats_packed`).

    python evaluate.py --chosen_snapshot PointDSC_3DMatch_release --root /data/3DMatch [--descriptor fcgf|fpfh] [--use_mutual]
    python evaluate.py --synthetic 8            # no dataset in this image: synthetic scene pairs, FPFH computed on the device

What it replaces, line by line (reference file:line):
  datasets/ThreeDMatch.py:226-231, :338-351   gt.log parsing, one entry per fragment pair           -> read_gt_log / list_pairs
  datasets/ThreeDMatch.py:240-258             fragment key points + descriptors from *.npz          -> load_fragment
  datasets/ThreeDMatch.py:261-267             gt_trans = inverse of the logged target->source pose  -> list_pairs
  datasets/ThreeDMatch.py:283-308             matching, labels, centred corr_pos                    -> match() + gt_labels()
  evaluation/test_3DMatch.py:38-54            .cuda() + model(data)                                 -> model(data) on device tensors
  evaluation/test_3DMatch.py:83-101           TransformationLoss / ClassificationLoss per pair      -> eval_stats (one launch, no sync)
  evaluation/test_3DMatch.py:139-172          scene-level and pair-level summary                    -> summarise
  evaluation/test_3DMatch.py:59-77            --solver RANSAC: open3d correspondence RANSAC      -> pointdsc_b200.ransac (row f6)
  evaluation/test_3DMatch.py:79-80            --use_icp: icp_refine (open3d registration_icp, r 0.10) -> pointdsc_b200.icp (row f5)
  baseline_scripts/baseline_3DMatch.py:19-53  --method SM: the spectral-matching baseline in place of the network
                                                                                         -> pointdsc_b200.spectral
The statistics of ALL pairs stay on the device and are read once at the end.  With --solver RANSAC the rows the network labelled
as inliers go through correspondence RANSAC on the device (3-point samples, 5,000 iterations, max correspondence distance = the
snapshot's inlier_threshold), whose transform and inliers replace the network's; with --use_icp the transform is then refined by
point-to-point ICP over the pair's correspondence key points (max correspondence distance 0.10 for every snapshot, as the reference
passes it).  Both run after the forward and before the statistics, inside the model time, in the drivers' order.  With
--method SM the spectral-matching baseline (inlier threshold = the snapshot's) takes the forward's place, inside the model time;
no network is loaded, and the baseline script has neither RANSAC nor ICP, so --method SM refuses both.  The FCGF
network is out of scope (DESIGN.md section 8); the FCGF descriptors of the reference's data set are plain *.npz files and work."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref")
GOLDEN = {"PointDSC_3DMatch_release": "snapshot_3dmatch.npz", "PointDSC_KITTI_release": "snapshot_kitti.npz"}
# snapshot/<name>/config.json of the reference: the fields the evaluation drivers read (evaluation/test_3DMatch.py:215-224)
CONFIG = {"PointDSC_3DMatch_release": dict(descriptor="fcgf", in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1,
                                           inlier_threshold=0.10, sigma_d=0.10, k=40, re_thre=15.0, te_thre=30.0, downsample=0.05,
                                           use_mutual=False),
          "PointDSC_KITTI_release": dict(descriptor="fcgf", in_dim=6, num_layers=12, num_channels=128, num_iterations=10, ratio=0.1,
                                         inlier_threshold=0.6, sigma_d=1.2, k=40, re_thre=5.0, te_thre=60.0, downsample=0.30,
                                         use_mutual=False)}
SCENES_3DMATCH = ["7-scenes-redkitchen", "sun3d-home_at-home_at_scan1_2013_jan_1", "sun3d-home_md-home_md_scan9_2012_sep_30",
                  "sun3d-hotel_uc-scan3", "sun3d-hotel_umd-maryland_hotel1", "sun3d-hotel_umd-maryland_hotel3",
                  "sun3d-mit_76_studyroom-76-1studyroom2", "sun3d-mit_lab_hj-lab_hj_tea_nov_2_2012_scan1_erika"]
# columns of the returned table: the reference's stats row (evaluation/test_3DMatch.py:26-27) + rmse
COLUMNS = ("success", "re_deg", "te_cm", "gt_inliers", "gt_inlier_ratio", "kept_gt_inliers", "precision", "recall", "f1",
           "model_time_s", "data_time_s", "scene", "rmse")


def load_config(name):
    cfg = dict(CONFIG[name])
    path = os.path.join(REF, "snapshot", name, "config.json")
    if os.path.exists(path):                     # the reference's own file where it has been installed (oracle/_ref)
        ref = json.load(open(path))
        cfg.update({k: ref[k] for k in cfg if k in ref})
    return cfg


def read_gt_log(path):
    """{'i_j': 4x4 float64} from a 3DMatch `gt.log` (datasets/ThreeDMatch.py:338-351): a header line `i \\t j \\t n` followed
    by the four rows of the pose that maps fragment j (target) into fragment i (source)."""
    with open(path) as f:
        lines = [ln for ln in f.read().splitlines() if ln.strip()]
    out = {}
    for i in range(0, len(lines) - 4, 5):
        head = lines[i].split()
        out[f"{int(head[0])}_{int(head[1])}"] = np.array([[float(x) for x in lines[i + r].split()] for r in range(1, 5)])
    return out


def list_pairs(root, scene):
    """[(src_id, tgt_id, gt_trans src->tgt)] of one scene, in gt.log order (datasets/ThreeDMatch.py:226-231, :261-267)."""
    log = read_gt_log(os.path.join(root, "gt_result", f"{scene}-evaluation", "gt.log"))
    return [(int(k.split("_")[0]), int(k.split("_")[1]), np.linalg.inv(v)) for k, v in log.items()]


def to_device(array, device):
    """A host array on the device without waiting for the stream: staged in page-locked memory and copied asynchronously, so
    that loading the next pair does not wait for the forward already enqueued (a copy from pageable memory would)."""
    t = torch.from_numpy(array)
    return t.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else t.to(device)


def load_fragment(root, scene, idx, descriptor, device):
    """Key points [n,3] float32 and descriptors [n,D] of `cloud_bin_{idx}_{descriptor}.npz` (datasets/ThreeDMatch.py:240-258);
    FPFH rows are normalised as the reference does it, x / (||x|| + 1e-6) in float64."""
    z = np.load(os.path.join(root, "fragments", scene, f"cloud_bin_{idx}_{descriptor}.npz"))
    xyz = to_device(np.ascontiguousarray(z["xyz"], dtype=np.float32), device)
    feat = to_device(np.ascontiguousarray(z["feature"]), device)
    if descriptor == "fpfh":
        feat = feat.double()
        feat = feat / (feat.norm(dim=1, keepdim=True) + 1e-6)
    else:
        feat = feat.float()
    return xyz, feat


def gt_labels(data, gt_trans, inlier_threshold):
    """labels = ||T_gt x_i - y_i|| < inlier_threshold over the putative correspondences (datasets/ThreeDMatch.py:293-297)."""
    src, tgt = data["src_keypts"][0], data["tgt_keypts"][0]
    warped = src @ gt_trans[:3, :3].T + gt_trans[:3, 3]
    return ((warped - tgt).pow(2).sum(-1).sqrt() < inlier_threshold).float()[None]


def build_model(snapshot, cfg, device, precision=None, batch_invariant=False):
    from pointdsc_b200 import PointDSC
    kw = {"batch_invariant": batch_invariant}
    if precision is not None:
        kw["precision"] = precision
    model = PointDSC(in_dim=cfg["in_dim"], num_layers=cfg["num_layers"], num_channels=cfg["num_channels"],
                     num_iterations=cfg["num_iterations"], ratio=cfg["ratio"], sigma_d=cfg["sigma_d"], k=cfg["k"],
                     nms_radius=cfg["inlier_threshold"], **kw)                           # evaluation/test_3DMatch.py:215-224
    pkl = os.path.join(REF, "snapshot", snapshot, "models", "model_best.pkl")
    state = None
    if os.path.exists(pkl):
        try:
            state = torch.load(pkl, map_location="cpu")                                  # the released file itself
        except Exception:
            state = None
    if state is None:
        z = np.load(os.path.join(ROOT, "tests", "golden", GOLDEN[snapshot]))             # its tensors, key for key
        state = {k: torch.from_numpy(z[k]) for k in z.files}
    miss = model.load_state_dict(state, strict=False)
    assert miss.missing_keys == [], miss
    return model.to(device).eval()


def synthetic_pairs(count, device, voxel):
    """`count` pairs of synthetic indoor-like fragments (pointdsc_b200.synth_scene) with FPFH descriptors computed on the device
    (row f2): yields (scene index, (src xyz, src desc), (tgt xyz, tgt desc), gt_trans)."""
    from pointdsc_b200.descriptors import fpfh_descriptors
    from pointdsc_b200.synth_scene import rigid, scene
    for p in range(count):
        R, t = rigid(100 + p)
        src = torch.from_numpy(scene(60000, seed=2 * p, layout_seed=20 + p)).to(device)
        tgt = torch.from_numpy((scene(60000, seed=2 * p + 1, layout_seed=20 + p).astype(np.float64) @ R.T + t).astype(np.float32)).to(device)
        gt = np.eye(4)
        gt[:3, :3], gt[:3, 3] = R, t
        yield p % 2, fpfh_descriptors(src, voxel), fpfh_descriptors(tgt, voxel), gt


def dataset_pairs(root, scenes, descriptor, device):
    for si, scene in enumerate(scenes):
        for src_id, tgt_id, gt in list_pairs(root, scene):
            yield si, load_fragment(root, scene, src_id, descriptor, device), load_fragment(root, scene, tgt_id, descriptor, device), gt


class SpectralMatching:
    """The spectral-matching baseline with the two calls `evaluate` makes of a model: `model(data)` per pair and
    `forward_packed` per group (baseline_scripts/baseline_3DMatch.py:19-53, `SM(corr, src_keypts, tgt_keypts, args)`)."""

    def __init__(self, inlier_threshold):
        self.inlier_threshold = float(inlier_threshold)

    def __call__(self, data):
        from pointdsc_b200.spectral import spectral_matching
        trans, labels = spectral_matching(data["corr_pos"], data["src_keypts"], data["tgt_keypts"], self.inlier_threshold)
        return {"final_trans": trans, "final_labels": labels}

    def forward_packed(self, corr_pos, src_keypts, tgt_keypts, offsets, d_offsets=None):
        from pointdsc_b200.spectral import spectral_matching_packed
        trans, labels = spectral_matching_packed(corr_pos, src_keypts, tgt_keypts, offsets, d_offsets=d_offsets,
                                                 inlier_threshold=self.inlier_threshold)
        return {"final_trans": trans, "final_labels": labels}


@torch.no_grad()
def evaluate(model, pairs, cfg, use_mutual=False, device="cuda", batch_size=1, use_icp=False, solver="SVD"):
    """The loop of evaluation/test_3DMatch.py:21-103 over an iterable of (scene index, (src xyz, src desc), (tgt xyz, tgt desc),
    gt_trans): returns a [pairs, 13] float64 array, columns = COLUMNS.
    batch_size 1: per pair `match`, labels, `model(data)` and `eval_stats`; the only read from the device inside the loop is the
    correspondence count of `match` with the mutual check (it fixes the tensor shapes).
    batch_size P > 1: every P pairs (each with its own number of correspondences) are matched in ONE call (`match_many`),
    labelled, run through ONE mixed-size forward (`PointDSC.forward_packed`) and scored by ONE `eval_stats_packed`, and nothing
    is read from the device inside the loop (with the mutual check: the group's P + 1 offsets, once).  The model-time column
    of a pair is then its group's device time divided by the group's size, and its data-time column its own loading time plus
    its share of the group's matching.  A model without `forward_packed` that offers `forward_many` (a wrapper or stand-in
    with the mixed-size interface only) is grouped pair by pair instead: `match`, labels, one `forward_many` per group and
    `eval_stats` per pair.
    solver "RANSAC": the forward's labels and transform are replaced by correspondence RANSAC's over the rows the network kept
    (evaluation/test_3DMatch.py:59-77, max correspondence distance cfg["inlier_threshold"]), on the device, before ICP and the
    statistics and inside the model-time events: `ransac_refine` per pair, one `ransac_packed` per packed group.
    use_icp: the transform is then refined on the device, also inside the model-time events (evaluation/test_3DMatch.py:79-80):
    `icp_refine` per pair, one `icp_refine_packed` per packed group."""
    from pointdsc_b200.frontend import match, match_many
    from pointdsc_b200.metrics import eval_stats, eval_stats_packed
    rows, scene_ids, data_s, events = [], [], [], []
    packed = batch_size > 1 and hasattr(model, "forward_packed")
    group = []          # pairs waiting for the group: packed ((src xyz, src desc), (tgt xyz, tgt desc), gt), else (data, gt_t, labels)
    if solver not in ("SVD", "RANSAC"):
        raise ValueError(f"solver must be SVD or RANSAC, got {solver!r}")
    if use_icp:
        from pointdsc_b200 import icp
    if solver == "RANSAC":
        from pointdsc_b200 import ransac

    def refine(data, res):
        """(trans, labels) of a pair after the drivers' post-steps: RANSAC, then ICP."""
        trans, labels = res["final_trans"], res["final_labels"]
        if solver == "RANSAC":
            trans, labels = ransac.ransac_refine(data["src_keypts"], data["tgt_keypts"], labels, cfg["inlier_threshold"])
        if use_icp:
            trans = icp.icp_refine(data["src_keypts"], data["tgt_keypts"], trans)
        return trans, labels

    def run_pair_group():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        results = model.forward_many([g[0] for g in group])
        refined = [refine(data, res) for (data, _, _), res in zip(group, results)]
        e1.record()
        for (data, gt_t, labels), (tr, pred) in zip(group, refined):
            rows.append(eval_stats(tr, gt_t[None], data["src_keypts"], data["tgt_keypts"], pred, labels, re_thre=cfg["re_thre"],
                                   te_thre=cfg["te_thre"]))
            events.append((e0, e1, len(group)))
        group.clear()

    def run_packed_group():
        t0 = time.perf_counter()
        m = match_many([(s[1], t[1], s[0], t[0]) for s, t, _ in group], use_mutual=use_mutual)
        off = m["offsets"]
        gts = to_device(np.stack([np.asarray(gt, dtype=np.float32) for _, _, gt in group]), device)
        labels = torch.cat([gt_labels({"src_keypts": m["src_keypts"][None, a:b], "tgt_keypts": m["tgt_keypts"][None, a:b]},
                                      gts[p], cfg["inlier_threshold"])[0] for p, (a, b) in enumerate(zip(off[:-1], off[1:]))])
        share = (time.perf_counter() - t0) / len(group)
        for p in range(len(group)):
            data_s[len(data_s) - len(group) + p] += share
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = model.forward_packed(m["corr_pos"], m["src_keypts"], m["tgt_keypts"], off, d_offsets=m["d_offsets"])
        trans, pred = res["final_trans"], res["final_labels"]
        if solver == "RANSAC":
            trans, pred = ransac.ransac_packed(m["src_keypts"], m["tgt_keypts"], pred, off, d_offsets=m["d_offsets"],
                                               max_correspondence_distance=cfg["inlier_threshold"])
        if use_icp:
            trans = icp.icp_refine_packed(m["src_keypts"], m["tgt_keypts"], trans, off, d_offsets=m["d_offsets"])
        e1.record()
        rows.append(eval_stats_packed(trans, gts, m["src_keypts"], m["tgt_keypts"], pred, labels, off,
                                      d_offsets=m["d_offsets"], re_thre=cfg["re_thre"], te_thre=cfg["te_thre"]))
        events.extend([(e0, e1, len(group))] * len(group))
        group.clear()

    run_group = run_packed_group if packed else run_pair_group
    t_data = time.perf_counter()
    for si, src, tgt, gt in pairs:
        scene_ids.append(si)
        if packed:
            data_s.append(time.perf_counter() - t_data)
            group.append((src, tgt, gt))
            if len(group) == batch_size:
                run_group()
            t_data = time.perf_counter()
            continue
        (src_xyz, src_desc), (tgt_xyz, tgt_desc) = src, tgt
        data = match(src_desc, tgt_desc, src_xyz, tgt_xyz, use_mutual=use_mutual)
        gt_t = torch.from_numpy(np.asarray(gt, dtype=np.float32)).to(device)
        labels = gt_labels(data, gt_t, cfg["inlier_threshold"])
        data["testing"] = True
        data_s.append(time.perf_counter() - t_data)
        if batch_size > 1:
            group.append((data, gt_t, labels))
            if len(group) == batch_size:
                run_group()
            t_data = time.perf_counter()
            continue
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = model(data)
        trans, pred = refine(data, res)
        e1.record()
        rows.append(eval_stats(trans, gt_t[None], data["src_keypts"], data["tgt_keypts"], pred, labels, re_thre=cfg["re_thre"],
                               te_thre=cfg["te_thre"]))
        events.append((e0, e1, 1))
        t_data = time.perf_counter()
    if group:
        run_group()
    if not rows:
        return np.zeros((0, len(COLUMNS)))
    dev_stats = torch.cat(rows, 0).double().cpu().numpy()          # the one read of the statistics
    out = np.zeros((len(dev_stats), len(COLUMNS)))
    out[:, :9] = dev_stats[:, :9]
    out[:, 9] = [a.elapsed_time(b) * 1e-3 / n for a, b, n in events]
    out[:, 10] = data_s
    out[:, 11] = scene_ids
    out[:, 12] = dev_stats[:, 9]
    return out


def summarise(stats, scene_names=None, log=print):
    """The reference's summary (evaluation/test_3DMatch.py:139-172): per scene, scene-level average, pair-level average; RE / TE are
    averaged over the successfully registered pairs only."""
    if len(stats) == 0:
        log("no pairs")
        return {}
    scenes = sorted(set(int(s) for s in stats[:, 11]))
    vals = []
    for s in scenes:
        st = stats[stats[:, 11] == s]
        v = st.mean(0)
        ok = st[st[:, 0] == 1]
        v[1], v[2] = (ok[:, 1].mean(), ok[:, 2].mean()) if len(ok) else (float("nan"), float("nan"))
        vals.append(v)
        name = scene_names[s] if scene_names else f"{s}th"
        log(f"Scene {name}: Reg Recall={v[0] * 100:.2f}%  Mean RE={v[1]:.2f}  Mean TE={v[2]:.2f}  Mean Precision={v[6] * 100:.2f}%  "
            f"Mean Recall={v[7] * 100:.2f}%  Mean F1={v[8] * 100:.2f}%")
    avg = np.nanmean(np.stack(vals), 0)
    log(f"All {len(scenes)} scenes, Mean Reg Recall={avg[0] * 100:.2f}%, Mean Re={avg[1]:.2f}, Mean Te={avg[2]:.2f}")
    allp = stats.mean(0)
    ok = stats[stats[:, 0] == 1]
    re, te = (ok[:, 1].mean(), ok[:, 2].mean()) if len(ok) else (float("nan"), float("nan"))
    log("*" * 40)
    log(f"All {len(stats)} pairs, Mean Reg Recall={allp[0] * 100:.2f}%, Mean Re={re:.2f}, Mean Te={te:.2f}")
    log(f"\tInput:  Mean Inlier Num={allp[3]:.2f}(ratio={allp[4] * 100:.2f}%)")
    log(f"\tOutput: Mean Inlier Num={allp[5]:.2f}(precision={allp[6] * 100:.2f}%, recall={allp[7] * 100:.2f}%, f1={allp[8] * 100:.2f}%)")
    log(f"\tMean model time: {allp[9] * 1e3:.2f}ms, Mean data time: {allp[10] * 1e3:.2f}ms")
    return {"pairs": int(len(stats)), "reg_recall": float(allp[0]), "mean_re_deg": float(re), "mean_te_cm": float(te),
            "precision": float(allp[6]), "recall": float(allp[7]), "f1": float(allp[8]), "model_ms": float(allp[9] * 1e3),
            "scene_recall": float(avg[0])}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--chosen_snapshot", default="PointDSC_3DMatch_release", choices=sorted(GOLDEN))
    ap.add_argument("--root", default="/data/3DMatch", help="data set root in the reference's layout (fragments/, gt_result/)")
    ap.add_argument("--descriptor", default=None, choices=["fcgf", "fpfh"])
    ap.add_argument("--use_mutual", action="store_true")
    ap.add_argument("--synthetic", type=int, default=0, help="evaluate on this many synthetic scene pairs instead of --root")
    ap.add_argument("--precision", default=None, help="fp16x3 (default) | fp32 | bf16x3 | bf16")
    ap.add_argument("--save_npy", default=None, help="write the [pairs, 13] statistics table here")
    ap.add_argument("--batch_size", type=int, default=1,
                    help="pairs per group: > 1 matches, runs and scores every group of pairs (of different sizes) in one call each")
    ap.add_argument("--batch_invariant", action="store_true",
                    help="every pair's result independent of --batch_size and of the GPU's SM count (PointDSC batch_invariant)")
    ap.add_argument("--use_icp", action="store_true",
                    help="refine every transform by point-to-point ICP on the device (max correspondence distance 0.10)")
    ap.add_argument("--solver", default="SVD", choices=["SVD", "RANSAC"],
                    help="RANSAC: replace the network's transform and labels by correspondence RANSAC over the rows it kept "
                         "(on the device, 5,000 iterations, max correspondence distance = the snapshot's inlier_threshold)")
    ap.add_argument("--method", default="PointDSC", choices=["PointDSC", "SM"],
                    help="SM: the spectral-matching baseline (baseline_scripts/baseline_3DMatch.py) in place of the network, "
                         "with the snapshot's inlier_threshold; no RANSAC, no ICP")
    return ap.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    cfg = load_config(args.chosen_snapshot)
    descriptor = args.descriptor or cfg["descriptor"]
    if args.method == "SM":
        if args.solver != "SVD" or args.use_icp:
            sys.exit("--method SM runs the spectral-matching baseline alone: it takes neither --solver RANSAC nor --use_icp")
        model = SpectralMatching(cfg["inlier_threshold"])
    else:
        model = build_model(args.chosen_snapshot, cfg, "cuda", args.precision, args.batch_invariant)
    if args.synthetic > 0:
        pairs, names = synthetic_pairs(args.synthetic, "cuda", 1.6 * cfg["downsample"]), ["synthetic-a", "synthetic-b"]
    else:
        names = [s for s in SCENES_3DMATCH if os.path.isdir(os.path.join(args.root, "fragments", s))]
        if not names:
            sys.exit(f"no 3DMatch test scene under {args.root}/fragments (this image has no data set: try --synthetic 8)")
        pairs = dataset_pairs(args.root, names, descriptor, "cuda")
    if args.batch_size < 1:
        sys.exit("--batch_size must be >= 1")
    stats = evaluate(model, pairs, cfg, use_mutual=args.use_mutual or cfg["use_mutual"], batch_size=args.batch_size,
                     use_icp=args.use_icp, solver=args.solver)
    summary = summarise(stats, names)
    if args.save_npy:
        np.save(args.save_npy, stats)
    return stats, summary


if __name__ == "__main__":
    main()
