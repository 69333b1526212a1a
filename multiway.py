#!/usr/bin/env python
"""The reference's multiway registration experiment (`multiway/test_multi_ate.py`) with every per-pair step on the H100: the
absolute trajectory error (ATE) of a scene's fragments after pairwise registration and pose-graph optimisation.

    python multiway.py --root /data/Augmented_ICL-NUIM [--scenes livingroom1-simulated ...] [--use_icp false]
    python multiway.py --synthetic 8           # no data set in this image: 8 synthetic views of one room, FPFH on the device

Per scene, over every pair i < j in the reference's order (test_multi_ate.py:88-180):
  odometry pairs (j = i + 1)   local_refinement from the fragment's odometry  -> one pointdsc_b200.multiway.multi_scale_icp_packed
  loop closures                matching, model(data) and the information       -> per --batch_size group: frontend.match_many,
                               matrix of the correspondence key points (0.07)     PointDSC.forward_packed, information_matrix_packed
  edge pruning                 info[5,5] / min(Ns, Nt) < 0.30 or trace(T) == 4  -> on the host, after ONE read of the scene's results
  global_optimization          open3d's Levenberg-Marquardt, line process       -> pointdsc_b200.multiway.global_optimization (host)
  --use_icp (default true)     local_refinement of every surviving edge         -> one multi_scale_icp_packed over all of them
The graphs go to {out_dir}/{scene}_fpfh_0/_1/_2.json in open3d's format; the ATE (test_multi_ate.py:260-288) is printed per scene.

Inputs follow the reference's layout: {root}/{scene}/fragments/fragment_XXX_fpfh.npz (xyz + FPFH, as cal_fpfh.py writes them),
fragment_XXX.npy (the ground-truth pose) and fragment_optimized_XXX.json (the odometry initialisation: the inverse of the last
node's pose).  The forward accepts at most 16,384 correspondences per set, so --num_node (the reference's 20,000) defaults to
16,384 and larger values are refused; fragments above it are subsampled with a seeded generator (the reference's
np.random.choice was unseeded).  With --synthetic K the odometry initialisation is the ground-truth step perturbed by a few
degrees and centimetres."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from pointdsc_b200 import frontend  # noqa: E402
from pointdsc_b200 import multiway as mw  # noqa: E402

SCENES = ["livingroom1-simulated", "livingroom2-simulated", "office1-simulated", "office2-simulated"]
MAX_NUM_NODE = 16384            # the forward's largest set
VOXEL = 0.05                    # cal_fpfh.py's key-point voxel
DISTANCE = 0.05 * 1.4           # max correspondence distance of the loop closures' information and of the optimisation


def scene_pairs(K):
    """Every pair i < j of K fragments in the reference's order (sorted by (i, j)): (odometry pairs, loop closures, all)."""
    pairs = [(i, j) for i in range(K) for j in range(i + 1, K)]
    return [p for p in pairs if p[1] == p[0] + 1], [p for p in pairs if p[1] != p[0] + 1], pairs


def subsample(n, num_node, seed, i, j, side):
    """The reference's key-point selection (datasets/Redwood.py:146-151), with a generator seeded by the pair."""
    if n <= num_node:
        return None
    return np.sort(np.random.default_rng([seed, i, j, side]).choice(n, num_node, replace=False))


def keep_loop_closure(trans, info, n):
    """The driver's test (test_multi_ate.py:130): drop the edge when info[5,5] / min(Ns, Nt) < 0.30 or trace(T) == 4."""
    return not (info[5, 5] / n < 0.30 or np.float32(np.trace(np.asarray(trans, np.float32))) == 4.0)


def perturb(T, rng, deg=3.0, cm=3.0):
    """T moved by a random rotation of `deg` degrees and a translation of `cm` centimetres."""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = np.deg2rad(deg)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    D = np.eye(4)
    D[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    shift = rng.normal(size=3)
    D[:3, 3] = cm / 100.0 * shift / np.linalg.norm(shift)
    return D @ T


def synthetic_scene(K, seed, device):
    """K synthetic views (pointdsc_b200.synth_scene.fragment_sequence) with FPFH key points computed on the device at VOXEL."""
    from pointdsc_b200.descriptors import fpfh_descriptors_many
    from pointdsc_b200.synth_scene import fragment_sequence
    views = fragment_sequence(K, seed)
    kp, feat, off, _ = fpfh_descriptors_many([torch.from_numpy(v).to(device) for v, _ in views], VOXEL, normalise=True)
    gt = [pose for _, pose in views]
    rng = np.random.default_rng(seed + 1)
    inits = [perturb(np.linalg.inv(gt[i + 1]) @ gt[i], rng) for i in range(K - 1)]
    return {"xyz": [kp[a:b] for a, b in zip(off[:-1], off[1:])], "feat": [feat[a:b] for a, b in zip(off[:-1], off[1:])],
            "gt": gt, "odometry_init": inits}


def dataset_scene(root, scene, device):
    """A scene in the reference's layout (datasets/Redwood.py:57-75, test_multi_ate.py:108-111)."""
    frag = os.path.join(root, scene, "fragments")
    K = 1 + max(int(f.split("_")[1]) for f in os.listdir(frag) if f.endswith("_fpfh.npz"))
    xyz, feat, gt, inits = [], [], [], []
    for k in range(K):
        z = np.load(os.path.join(frag, f"fragment_{k:03d}_fpfh.npz"))
        xyz.append(torch.from_numpy(np.ascontiguousarray(z["xyz"], np.float32)).to(device))
        f = torch.from_numpy(np.ascontiguousarray(z["feature"], np.float64)).to(device)
        feat.append(f / (f.norm(dim=1, keepdim=True) + 1e-6))
        gt.append(np.load(os.path.join(frag, f"fragment_{k:03d}.npy")))
        if k + 1 < K:
            g = mw.read_pose_graph(os.path.join(frag, f"fragment_optimized_{k:03d}.json"))
            inits.append(np.linalg.inv(g.nodes[-1]))
    return {"xyz": xyz, "feat": feat, "gt": gt, "odometry_init": inits}


def graph_from_edges(results):
    """The reference's graph of a list of (i, j, T, info) in order: odometry edges chain the nodes (pose = inverse of the
    accumulated odometry) and are certain, the others are uncertain loop closures."""
    g = mw.PoseGraph([np.eye(4)], [])
    odometry = np.eye(4)
    for i, j, T, info in results:
        T = np.asarray(T, np.float64)
        if j == i + 1:
            odometry = T @ odometry
            g.nodes.append(np.linalg.inv(odometry))
        g.edges.append(mw.PoseGraphEdge(i, j, T, np.asarray(info, np.float64), uncertain=j != i + 1))
    return g


@torch.no_grad()
def register_scene(model, data, batch_size=8, num_node=MAX_NUM_NODE, seed=0, log=print):
    """The scene's pose graph before optimisation (test_multi_ate.py:88-150): one grouped ICP call for the odometry pairs, one
    match / forward / information call per group of loop closures, one read of every result at the end."""
    K = len(data["xyz"])
    odo, loops, pairs = scene_pairs(K)
    dev = data["xyz"][0].device
    inits = torch.from_numpy(np.array([data["odometry_init"][i] for i, _ in odo], np.float32)).to(dev)
    T_odo, I_odo = mw.multi_scale_icp_packed(data["xyz"], odo, inits)
    T_loop, I_loop, sizes = [], [], []
    for g in range(0, len(loops), batch_size):
        items = []
        for i, j in loops[g:g + batch_size]:
            si = subsample(int(data["xyz"][i].shape[0]), num_node, seed, i, j, 0)
            ti = subsample(int(data["xyz"][j].shape[0]), num_node, seed, i, j, 1)
            pick = lambda x, sel: x if sel is None else x[torch.from_numpy(sel).to(dev)]  # noqa: E731
            items.append((pick(data["feat"][i], si), pick(data["feat"][j], ti), pick(data["xyz"][i], si), pick(data["xyz"][j], ti)))
        m = frontend.match_many(items)
        out = model.forward_packed(m["corr_pos"], m["src_keypts"], m["tgt_keypts"], m["offsets"], d_offsets=m["d_offsets"])
        info = mw.information_matrix_packed(m["src_keypts"], m["tgt_keypts"], out["final_trans"], m["offsets"], m["offsets"],
                                            d_src_offsets=m["d_offsets"], d_tgt_offsets=m["d_offsets"],
                                            max_correspondence_distance=DISTANCE)
        T_loop.append(out["final_trans"])
        I_loop.append(info)
        sizes += [b - a for a, b in zip(m["offsets"][:-1], m["offsets"][1:])]
    # the one read of the scene: every transform and information matrix
    T_odo, I_odo = T_odo.cpu().numpy(), I_odo.cpu().numpy()
    if loops:
        T_loop, I_loop = torch.cat(T_loop).cpu().numpy(), torch.cat(I_loop).cpu().numpy()
    results, k_odo, k_loop = [], 0, 0
    for i, j in pairs:
        if j == i + 1:
            results.append((i, j, T_odo[k_odo], I_odo[k_odo]))
            k_odo += 1
        else:
            if keep_loop_closure(T_loop[k_loop], I_loop[k_loop], sizes[k_loop]):
                results.append((i, j, T_loop[k_loop], I_loop[k_loop]))
            k_loop += 1
    return graph_from_edges(results)


@torch.no_grad()
def refine_edges(data, graph):
    """test_multi_ate.py:170-205: local_refinement of every edge of `graph` from its transform, in one grouped call, and the
    graph rebuilt from the refined edges."""
    dev = data["xyz"][0].device
    pairs = [(e.source, e.target) for e in graph.edges]
    inits = torch.from_numpy(np.array([e.transformation for e in graph.edges], np.float32)).to(dev)
    T, info = mw.multi_scale_icp_packed(data["xyz"], pairs, inits)
    T, info = T.cpu().numpy(), info.cpu().numpy()
    return graph_from_edges([(i, j, T[k], info[k]) for k, (i, j) in enumerate(pairs)])


def optimise(graph, log):
    log(f"Before optimization {len(graph.nodes)} nodes {len(graph.edges)} edges")
    g = mw.global_optimization(graph, max_correspondence_distance=DISTANCE, edge_prune_threshold=0.25, preference_loop_closure=20.0,
                               reference_node=0)
    log(f"After optimization {len(g.nodes)} nodes {len(g.edges)} edges")
    return g


def run_scene(model, data, prefix, use_icp=True, batch_size=8, num_node=MAX_NUM_NODE, seed=0, log=print):
    """One scene end to end; writes {prefix}_0/_1(/_2).json and returns (final graph, ATE in cm)."""
    g0 = register_scene(model, data, batch_size, num_node, seed, log)
    mw.write_pose_graph(prefix + "_0.json", g0)
    g = optimise(g0, log)
    mw.write_pose_graph(prefix + "_1.json", g)
    if use_icp:
        g = optimise(refine_edges(data, g), log)
        mw.write_pose_graph(prefix + "_2.json", g)
    if len(g.nodes) != len(data["gt"]):
        raise RuntimeError(f"the graph has {len(g.nodes)} nodes for {len(data['gt'])} fragments")
    ate = mw.trajectory_ate(data["gt"], g.nodes)
    log(f"Mean Absolute Trajectory Error: {ate:.2f}cm")
    return g, ate


def _bool(s):
    if s.lower() in ("1", "true", "yes", "on"):
        return True
    if s.lower() in ("0", "false", "no", "off"):
        return False
    raise argparse.ArgumentTypeError(f"expected a boolean, got {s!r}")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--chosen_snapshot", default="PointDSC_3DMatch_release")
    ap.add_argument("--root", default="/data/Augmented_ICL-NUIM", help="data set root in the reference's layout")
    ap.add_argument("--scenes", nargs="*", default=None, help=f"scenes under --root (default: those of {SCENES} present)")
    ap.add_argument("--synthetic", type=int, default=0, help="run one synthetic scene of this many fragments instead of --root")
    ap.add_argument("--use_icp", type=_bool, default=True, help="refine every surviving edge by multi-scale ICP (default true)")
    ap.add_argument("--batch_size", type=int, default=8, help="loop-closure pairs per match / forward / information call")
    ap.add_argument("--num_node", type=int, default=MAX_NUM_NODE,
                    help=f"key points per fragment of a loop closure (at most {MAX_NUM_NODE}, the forward's largest set)")
    ap.add_argument("--seed", type=int, default=0, help="seed of the key-point subsampling and of the synthetic scene")
    ap.add_argument("--out_dir", default="multiway_out", help="where the pose graphs are written")
    args = ap.parse_args(argv)
    if args.num_node > MAX_NUM_NODE:
        ap.error(f"--num_node {args.num_node}: the forward accepts at most {MAX_NUM_NODE} correspondences per set")
    if args.num_node < 1 or args.batch_size < 1:
        ap.error("--num_node and --batch_size must be >= 1")
    if args.synthetic == 1 or args.synthetic < 0:
        ap.error("--synthetic needs at least two fragments")
    return args


def main(argv=None, model=None, log=print):
    args = parse_args(argv)
    if model is None:
        from evaluate import build_model, load_config
        model = build_model(args.chosen_snapshot, load_config(args.chosen_snapshot), "cuda")
    if args.synthetic:
        scenes = [("synthetic", lambda: synthetic_scene(args.synthetic, args.seed, "cuda"))]
    else:
        names = args.scenes or [s for s in SCENES if os.path.isdir(os.path.join(args.root, s, "fragments"))]
        if not names:
            sys.exit(f"no scene under {args.root} (this image has no data set: try --synthetic 8)")
        scenes = [(s, lambda s=s: dataset_scene(args.root, s, "cuda")) for s in names]
    os.makedirs(args.out_dir, exist_ok=True)
    ates = []
    for name, load in scenes:
        log(f"scene {name}")
        _, ate = run_scene(model, load(), os.path.join(args.out_dir, f"{name}_fpfh"), args.use_icp, args.batch_size, args.num_node,
                           args.seed, log)
        ates.append(ate)
    log(f"All {len(ates)} scene ATE(cm): {[round(a, 2) for a in ates]}")
    log(f"Mean ATE(cm): {np.mean(ates):.2f}cm")
    return ates


if __name__ == "__main__":
    main()
