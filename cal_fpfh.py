#!/usr/bin/env python
"""The reference's misc/cal_fpfh.py on the device, without open3d: FPFH files for every cloud of a data set.

    python cal_fpfh.py PATH [PATH ...] [--voxel_size 0.05] [--out DIR] [--max_points 4000000]

Inputs: every `*.ply` file and every `*.npz` file holding a `pcd` array under the given paths (files or directories, searched
recursively) — the one rule behind the reference's process_3dmatch (`threedmatch/*.npz`), process_3dmatch_test
(`fragments/<scene>/*.ply`) and process_redwood (`<scene>/fragments/*.ply`).  For each input `<stem>.ply` / `<stem>.npz` it
writes `<stem>_fpfh.npz` with the reference's keys and dtypes: `points` (the cloud as read, float32), `xyz` (the voxel
down-sampled key points, float32) and `feature` (the raw FPFH, float32) — what `evaluate.py --descriptor fpfh` reads through
`evaluate.load_fragment`.  Files go next to their input, as in the reference, or with `--out DIR` into a mirror of the input
tree under DIR (data sets are often read-only).

Clouds go to the device in groups of at most `--max_points` points in all (at least one cloud per group), which bounds the
voxel scratch; each group takes one call per stage (`descriptors.fpfh_descriptors_many`), and the next group's files are read
on the host while the device works on the current one.  A cloud without points is skipped with a message, as in the reference."""
import argparse
import os
import sys
import zipfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def find_inputs(paths):
    """[(input file, the root its output path is taken relative to)] in a fixed (sorted) order."""
    found = []
    for path in paths:
        if os.path.isfile(path):
            found.append((path, os.path.dirname(path)))
            continue
        if not os.path.isdir(path):
            raise FileNotFoundError(path)
        for d, dirs, files in os.walk(path):
            dirs.sort()
            found += [(os.path.join(d, f), path) for f in sorted(files)]
    out = []
    for f, root in found:
        if f.endswith(".ply"):
            out.append((f, root))
        elif f.endswith(".npz"):
            with np.load(f) as z:
                if "pcd" in z.files:
                    out.append((f, root))
    return out


def output_path(src, root, out_dir=None, suffix="_fpfh.npz"):
    stem = os.path.splitext(src)[0] + suffix
    return stem if out_dir is None else os.path.join(out_dir, os.path.relpath(stem, root))


def read_cloud(path):
    """The cloud of one input as [n,3] float32 (misc/cal_fpfh.py: `np.load(path)['pcd']`, `o3d.io.read_point_cloud(path).points`)."""
    if path.endswith(".ply"):
        from pointdsc_b200.descriptors import read_ply
        return read_ply(path)
    with np.load(path) as z:
        return np.ascontiguousarray(z["pcd"], dtype=np.float32).reshape(-1, 3)


def cloud_size(path):
    """Points of one input from its header alone (the PLY header, the `pcd` array's .npy header)."""
    if path.endswith(".ply"):
        import ctypes as C
        from pointdsc_b200 import _capi
        n = C.c_int64(0)
        _capi.check(_capi.load().pdsc_read_ply(path.encode(), None, 0, C.byref(n)))
        return int(n.value)
    fmt = np.lib.format
    with zipfile.ZipFile(path) as z, z.open("pcd.npy") as f:
        version = fmt.read_magic(f)
        read_header = {(1, 0): fmt.read_array_header_1_0, (2, 0): fmt.read_array_header_2_0}.get(version)
        if read_header is not None:
            return int(np.prod(read_header(f)[0])) // 3
    return len(read_cloud(path))


def describe_on_device(clouds, voxel_size):
    """[(xyz [m,3] float32, raw FPFH [m,33] float32)] of a group of host clouds: one call per stage on the current device."""
    import torch
    from pointdsc_b200.descriptors import fpfh_descriptors_many
    dev = [torch.from_numpy(c).pin_memory().to("cuda", non_blocking=True) for c in clouds]
    kp, feat, off, _ = fpfh_descriptors_many(dev, voxel_size, normalise=False)
    kp, feat = kp.cpu().numpy(), feat.cpu().numpy().astype(np.float32)      # misc/cal_fpfh.py:34: fpfh_np.astype(np.float32)
    return [(kp[off[p]:off[p + 1]], feat[off[p]:off[p + 1]]) for p in range(len(clouds))]


def make_groups(sizes, max_points):
    """Consecutive index groups whose point counts sum to at most max_points (a larger cloud is a group of its own)."""
    groups, cur, total = [], [], 0
    for i, n in enumerate(sizes):
        if cur and total + n > max_points:
            groups.append(cur)
            cur, total = [], 0
        cur.append(i)
        total += n
    if cur:
        groups.append(cur)
    return groups


def _read_group(items):
    return [read_cloud(f) for f, _ in items]


def run(paths, voxel_size=0.05, out_dir=None, max_points=4_000_000, describe=describe_on_device, log=print, suffix="_fpfh.npz"):
    """Write `<stem><suffix>` (by default `<stem>_fpfh.npz`) for every input under `paths`, with `describe(clouds, voxel_size)`
    giving each group's (xyz, feature) pairs; returns the files written, in input order."""
    inputs = find_inputs(paths)
    groups = make_groups([cloud_size(f) for f, _ in inputs], max_points)
    written = []
    with ThreadPoolExecutor(max_workers=1) as reader:
        pending = reader.submit(_read_group, [inputs[i] for i in groups[0]]) if groups else None
        for g, idx in enumerate(groups):
            clouds = pending.result()
            if g + 1 < len(groups):      # read the next group's files while the device works on this one
                pending = reader.submit(_read_group, [inputs[i] for i in groups[g + 1]])
            keep = [k for k, c in enumerate(clouds) if len(c)]
            for k in set(range(len(clouds))) - set(keep):
                log(f"{inputs[idx[k]][0]} error: do not have any points.")
            results = describe([clouds[k] for k in keep], voxel_size) if keep else []
            for k, (xyz, feat) in zip(keep, results):
                src, root = inputs[idx[k]]
                dst = output_path(src, root, out_dir, suffix)
                os.makedirs(os.path.dirname(os.path.abspath(dst)), exist_ok=True)
                np.savez_compressed(dst, points=clouds[k].astype(np.float32), xyz=xyz.astype(np.float32),
                                    feature=feat.astype(np.float32))
                log(src, feat.shape)
                written.append(dst)
    return written


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("paths", nargs="+", help="input files or directories (searched recursively)")
    ap.add_argument("--voxel_size", type=float, default=0.05)
    ap.add_argument("--out", default=None, help="write into a mirror of the input tree under this directory")
    ap.add_argument("--max_points", type=int, default=4_000_000, help="points per device group, all clouds together")
    args = ap.parse_args(argv)
    run(args.paths, args.voxel_size, args.out, args.max_points)


if __name__ == "__main__":
    main()
