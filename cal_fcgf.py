#!/usr/bin/env python
"""The reference's misc/cal_fcgf.py on the device, without MinkowskiEngine: FCGF files for every cloud of a data set.

    python cal_fcgf.py PATH [PATH ...] --weights ResUNetBN2C-feat32-3dmatch-v0.05.pth [--voxel_size 0.05] [--out DIR]
                       [--max_points 1000000]

Inputs, output placement, grouping and the host read-ahead are cal_fpfh.py's (every `*.ply`, and every `*.npz` holding a `pcd`
array, under the given paths).  For each input `<stem>.ply` / `<stem>.npz` it writes `<stem>_fcgf.npz` with `points` (the
cloud as read), `xyz` (one point per occupied voxel, the voxel's first point) and `feature` (the 32-channel unit descriptor),
all float32 — what `evaluate.py --descriptor fcgf` reads through `evaluate.load_fragment`.  The weights are the reference's
released FCGF checkpoints (cal_fcgf.py:344-370): the 3DMatch ones at voxel 0.05, the KITTI ones at 0.30; the conv1 kernel size
is read from the file.  A group takes one pdsc_fcgf_packed call; its scratch is about 11 KB per input point, which
`--max_points` bounds."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import cal_fpfh  # noqa: E402

_models = {}


def describe_on_device(clouds, voxel_size, weights):
    """[(xyz [m,3] float32, FCGF [m,32] float32)] of a group of host clouds: one call on the current device."""
    import torch
    from pointdsc_b200.fcgf import fcgf_descriptors_many, model_from_checkpoint
    if weights not in _models:
        _models[weights] = model_from_checkpoint(weights)
    dev = [torch.from_numpy(c).pin_memory().to("cuda", non_blocking=True) for c in clouds]
    kp, feat, off, _ = fcgf_descriptors_many(_models[weights], dev, voxel_size)
    kp, feat = kp.cpu().numpy(), feat.cpu().numpy()
    return [(kp[off[p]:off[p + 1]], feat[off[p]:off[p + 1]]) for p in range(len(clouds))]


def run(paths, weights, voxel_size=0.05, out_dir=None, max_points=1_000_000, describe=describe_on_device, log=print):
    """Write `<stem>_fcgf.npz` for every input under `paths`; returns the files written, in input order."""
    return cal_fpfh.run(paths, voxel_size, out_dir, max_points, describe=lambda c, v: describe(c, v, weights), log=log,
                        suffix="_fcgf.npz")


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("paths", nargs="+", help="input files or directories (searched recursively)")
    ap.add_argument("--weights", required=True, help="a released FCGF checkpoint (ResUNetBN2C-feat32-*.pth)")
    ap.add_argument("--voxel_size", type=float, default=0.05)
    ap.add_argument("--out", default=None, help="write into a mirror of the input tree under this directory")
    ap.add_argument("--max_points", type=int, default=1_000_000, help="points per device group, all clouds together")
    args = ap.parse_args(argv)
    if not os.path.exists(args.weights):
        sys.exit(f"{args.weights} not found: the reference downloads the FCGF weights from "
                 "http://node2.chrischoy.org/data/projects/DGR/ResUNetBN2C-feat32-3dmatch-v0.05.pth (3DMatch, voxel 0.05) and "
                 "ResUNetBN2C-feat32-kitti-v0.3.pth (KITTI, voxel 0.30)")
    run(args.paths, args.weights, args.voxel_size, args.out, args.max_points)


if __name__ == "__main__":
    main()
