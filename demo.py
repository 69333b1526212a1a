#!/usr/bin/env python
"""BASELINE.json configs[0] on the H100: the reference's `demo_registration.py --descriptor fpfh` with every step after the file
read on the device and without open3d (reference demo_registration.py:37-44, :78-117).

    python demo.py [--chosen_snapshot PointDSC_3DMatch_release] [--pcd1 a.ply --pcd2 b.ply] [--descriptor fpfh]

Defaults: the reference's own demo clouds (copied unmodified into the git-ignored oracle/_ref/demo_data by
`__graft_entry__.build()` when POINTDSC_REFERENCE names a checkout of the reference).  Prints the estimated transformation and, instead of the reference's
open3d windows, how much of the source cloud lies on the target before and after it.

`--descriptor fcgf --fcgf_weights PATH` describes both clouds with the FCGF network on the device (pointdsc_b200.fcgf, the
reference's extract_fcgf_features, demo_registration.py:11-34) instead of FPFH: the 3DMatch snapshot pairs with the reference's
ResUNetBN2C-feat32-3dmatch-v0.05.pth (conv1 kernel 7, voxel 0.05), the KITTI snapshot with ResUNetBN2C-feat32-kitti-v0.3.pth
(kernel 5, voxel 0.30); the voxel is the snapshot's downsample.  The weights are not shipped."""
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
# snapshot/<name>/config.json of the reference (the fields the demo reads, demo_registration.py:78-87)
CONFIG = {"PointDSC_3DMatch_release": dict(downsample=0.05, inlier_threshold=0.10, sigma_d=0.10, k=40, ratio=0.1, num_iterations=10),
          "PointDSC_KITTI_release": dict(downsample=0.30, inlier_threshold=0.6, sigma_d=1.2, k=40, ratio=0.1, num_iterations=10)}


def load_config(name):
    path = os.path.join(REF, "snapshot", name, "config.json")
    cfg = dict(CONFIG[name])
    if os.path.exists(path):                    # the reference's own file where it has been installed
        ref = json.load(open(path))
        cfg.update({k: ref[k] for k in cfg if k in ref})
    return cfg


def coverage(src, tgt, radius, trans=None, chunk=4096):
    """Fraction of the source key points that have a target key point within `radius` after `trans` (what the reference shows
    in an open3d window, as a number)."""
    if trans is not None:
        src = src @ trans[:3, :3].T + trans[:3, 3]
    hit = 0
    for i in range(0, src.shape[0], chunk):
        hit += int((torch.cdist(src[i:i + chunk], tgt).min(dim=1).values < radius).sum())
    return hit / src.shape[0]


@torch.no_grad()
def register(pcd1, pcd2, snapshot="PointDSC_3DMatch_release", device="cuda", verbose=True, return_data=False, descriptor="fpfh",
             fcgf_weights=None):
    from pointdsc_b200 import PointDSC
    from pointdsc_b200.descriptors import fpfh_descriptors, read_ply
    from pointdsc_b200.frontend import match
    cfg = load_config(snapshot)
    z = np.load(os.path.join(ROOT, "tests", "golden", GOLDEN[snapshot]))
    model = PointDSC(in_dim=6, num_layers=12, num_channels=128, num_iterations=cfg["num_iterations"], ratio=cfg["ratio"],
                     sigma_d=cfg["sigma_d"], k=cfg["k"], nms_radius=cfg["inlier_threshold"]).to(device)   # as demo_registration.py:78-87
    miss = model.load_state_dict({k: torch.from_numpy(z[k]) for k in z.files}, strict=False)
    model.eval()
    t0 = time.perf_counter()
    clouds = [torch.from_numpy(read_ply(p)).to(device) for p in (pcd1, pcd2)]
    t1 = time.perf_counter()
    if descriptor == "fcgf":                                                        # demo_registration.py:11-34
        from pointdsc_b200.fcgf import fcgf_descriptors_many, model_from_checkpoint
        kp, feat, off, _ = fcgf_descriptors_many(model_from_checkpoint(fcgf_weights), clouds, cfg["downsample"])
        (src_pts, src_feat), (tgt_pts, tgt_feat) = ((kp[off[p]:off[p + 1]], feat[off[p]:off[p + 1]]) for p in range(2))
    else:
        (src_pts, src_feat), (tgt_pts, tgt_feat) = (fpfh_descriptors(c, cfg["downsample"]) for c in clouds)
    data = match(src_feat, tgt_feat, src_pts, tgt_pts, use_mutual=False)          # demo_registration.py:101-108
    data["testing"] = True
    res = model(data)                                                               # demo_registration.py:117
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    trans = res["final_trans"][0]
    out = {"vertices": [int(c.shape[0]) for c in clouds], "key_points": [int(src_pts.shape[0]), int(tgt_pts.shape[0])],
           "correspondences": int(data["corr_pos"].shape[1]), "inliers": int(res["final_labels"].sum()),
           "final_trans": trans.cpu().numpy(), "missing_keys": list(miss.missing_keys),
           "coverage_before": coverage(src_pts, tgt_pts, 2 * cfg["downsample"]),
           "coverage_after": coverage(src_pts, tgt_pts, 2 * cfg["downsample"], trans),
           "seconds_read": t1 - t0, "seconds_device": t2 - t1}
    if return_data:       # the network input and the labels, for the parity test against the CPU checker
        out["data"] = {k: v for k, v in data.items() if k != "testing"}
        out["final_labels"] = res["final_labels"]
    if verbose:
        print(miss)
        for k, v in out.items():
            if k not in ("data", "final_labels"):
                print(f"{k}:\n{v}" if k == "final_trans" else f"{k}: {v}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chosen_snapshot", default="PointDSC_3DMatch_release", choices=sorted(GOLDEN))
    ap.add_argument("--pcd1", default=os.path.join(REF, "demo_data", "cloud_bin_0.ply"))
    ap.add_argument("--pcd2", default=os.path.join(REF, "demo_data", "cloud_bin_1.ply"))
    ap.add_argument("--descriptor", default="fpfh", choices=["fcgf", "fpfh"])
    ap.add_argument("--fcgf_weights", default=None, help="the FCGF checkpoint --descriptor fcgf reads")
    ap.add_argument("--use_gpu", default="True")
    a = ap.parse_args()
    if a.descriptor == "fcgf" and not (a.fcgf_weights and os.path.exists(a.fcgf_weights)):
        kitti = a.chosen_snapshot == "PointDSC_KITTI_release"
        sys.exit(f"--descriptor fcgf needs --fcgf_weights PATH ({a.fcgf_weights} not found).  The reference downloads them from "
                 "http://node2.chrischoy.org/data/projects/DGR/ResUNetBN2C-feat32-"
                 + ("kitti-v0.3.pth (conv1 kernel 5, voxel 0.30)" if kitti else "3dmatch-v0.05.pth (conv1 kernel 7, voxel 0.05)"))
    if str(a.use_gpu).lower() in ("false", "0", "no") or not torch.cuda.is_available():
        sys.exit("pointdsc_b200 runs on an H100 only (there is no CPU fallback)")
    register(a.pcd1, a.pcd2, a.chosen_snapshot, descriptor=a.descriptor, fcgf_weights=a.fcgf_weights)


if __name__ == "__main__":
    main()
