"""Multiway registration (row f7): what multiway/test_multi_ate.py needs beyond matching and the forward.

Device side, a group of fragment pairs per call and nothing read back:
  * `icp_clouds_packed`: open3d 0.9's point-to-point `registration_icp` between two different clouds (pdsc_icp_clouds_packed);
  * `information_matrix_packed`: `get_information_matrix_from_point_clouds` (pdsc_information_matrix_packed);
  * `multi_scale_icp_packed`: the driver's `local_refinement` (voxel 0.05 / 0.025 / 0.0125, 50 / 30 / 14 iterations, distance
    0.07, then the information matrix at the last scale with r = voxel * 1.4).

Host side, float64 (a graph of tens of nodes; not a hot path):
  * `PoseGraph`, `read_pose_graph` / `write_pose_graph` in open3d's JSON layout;
  * `global_optimization`: open3d 0.9's `global_optimization` with `GlobalOptimizationLevenbergMarquardt`, the line process and
    edge pruning;
  * `trajectory_ate`: the driver's `align` (Kabsch fit of the node positions, RMSE in cm).

open3d is not part of the reference tree or of this image.  The device calls follow its published algorithms and are checked
against the float64 restatements under oracle/; the host code restates open3d 0.9 from memory (RECALLED, parity
unpinned).  The conventions it assumes:
  * JSON: {"class_name": "PoseGraph", "nodes": [{"class_name": "PoseGraphNode", "pose": 16 numbers}], "edges":
    [{"class_name": "PoseGraphEdge", "source_node_id", "target_node_id", "transformation": 16, "information": 36, "uncertain",
    "confidence"}], "version_major": 1, "version_minor": 0}, every matrix column-major (Eigen's storage order);
  * a node's pose maps the fragment into the world; an edge's transformation maps its source fragment into its target's;
  * misalignment of an edge: E = T_edge^-1 P_t^-1 P_s, e = (-E[1,2], E[0,2], -E[0,1], E[0,3], E[1,3], E[2,3]);
  * Jacobians: column i of J_s is that 6-vector of T_edge^-1 P_t^-1 G_i P_s, of J_t of -(that), G_i the se(3) generators in
    the order rotation x, y, z, translation x, y, z; an update delta of node n is P_n <- M(delta_n) P_n with
    M = [Rz(c) Ry(b) Rx(a) | (d, e, f)];
  * line process: weight w = preference_loop_closure * max_correspondence_distance^2 * mean over edges of info[5,5]; an uncertain
    edge's confidence and line process l = (w / (w + e^T Info e))^2, certain edges 1; residual sum l e^T Info e + w (sqrt(l) - 1)^2;
  * Levenberg-Marquardt with GlobalOptimizationConvergenceCriteria's defaults (100 iterations, 20 LM tries, relative increment,
    relative residual increment, right term and residual 1e-6, scale factors 1/3 and 2/3), lambda_0 = 1e-5 max diag(H), nu = 2;
  * global_optimization: optimise, drop uncertain edges whose confidence is not above edge_prune_threshold, optimise again, then
    move every pose by P_ref(before) P_ref(after)^-1 so the reference node keeps its pose.
"""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _capi


def _check_offsets(name: str, offsets: Sequence[int]) -> List[int]:
    offsets = [int(o) for o in offsets]
    if len(offsets) < 2 or offsets[0] != 0 or any(b <= a for a, b in zip(offsets[:-1], offsets[1:])):
        raise ValueError(f"{name} must start at 0 and increase by at least 1 per pair, got {offsets}")
    return offsets


def _pair_args(src, tgt, src_offsets, tgt_offsets, d_src_offsets, d_tgt_offsets, trans, what):
    if src.device.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.multiway runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    src_offsets = _check_offsets("src_offsets", src_offsets)
    tgt_offsets = _check_offsets("tgt_offsets", tgt_offsets)
    B = len(src_offsets) - 1
    if len(tgt_offsets) != B + 1:
        raise ValueError(f"src_offsets and tgt_offsets must have the same length, got {B + 1} and {len(tgt_offsets)}")
    for name, t, rows in (("src", src, src_offsets[-1]), ("tgt", tgt, tgt_offsets[-1])):
        if t.device != src.device or t.dim() != 2 or t.shape[1] != 3 or t.shape[0] < rows:
            raise ValueError(f"{name} must be [>= {rows},3] on {src.device}, got {tuple(t.shape)} on {t.device}")
    if tuple(trans.shape) != (B, 4, 4):
        raise ValueError(f"{what} must be [{B},4,4], got {tuple(trans.shape)}")
    dev = src.device
    h_src, d_src = _capi.offsets(src_offsets, d_src_offsets, dev)
    h_tgt, d_tgt = _capi.offsets(tgt_offsets, d_tgt_offsets, dev)
    s = src.to(torch.float32).contiguous()
    t = tgt.to(torch.float32).contiguous()
    return B, dev, s, t, trans.to(device=dev, dtype=torch.float32).contiguous(), h_src, d_src, h_tgt, d_tgt


def _ptr(x):
    return C.c_void_p(x.data_ptr()) if x is not None else None


@torch.no_grad()
def icp_clouds_packed(src: torch.Tensor, tgt: torch.Tensor, init: torch.Tensor, src_offsets: Sequence[int], tgt_offsets: Sequence[int],
                      d_src_offsets: Optional[torch.Tensor] = None, d_tgt_offsets: Optional[torch.Tensor] = None,
                      max_correspondence_distance: float = 0.07, max_iteration: int = 30, info: bool = False):
    """Point-to-point ICP of B pairs of different clouds in one call (pdsc_icp_clouds_packed).  Pair b's source is rows
    src_offsets[b]:src_offsets[b+1] of src, its target rows tgt_offsets[b]:tgt_offsets[b+1] of tgt; init [B,4,4].  The device
    offsets (uploaded when None) are what the kernel reads; they may describe fewer rows than the host ones, as a packed voxel
    down-sampling writes them (see the header).  Returns the refined [B,4,4] float32; with info=True also {'fitness' (kept /
    Ns), 'inlier_rmse', 'iterations', 'status'} as `icp.icp_refine_packed`.  Nothing is read back."""
    B, dev, s, t, init, h_src, d_src, h_tgt, d_tgt = _pair_args(src, tgt, src_offsets, tgt_offsets, d_src_offsets, d_tgt_offsets,
                                                                init, "init")
    lib, engine, stream = _capi.device_context(dev)
    out = torch.empty(B, 4, 4, dtype=torch.float32, device=dev)
    stats = torch.empty(2, B, dtype=torch.float64, device=dev) if info else None
    ints = torch.empty(2, B, dtype=torch.int32, device=dev) if info else None
    scratch = _capi.scratch(lib.pdsc_icp_clouds_packed_scratch_bytes(B, h_src, h_tgt), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_icp_clouds_packed(engine, B, h_src, h_tgt, _ptr(d_src), _ptr(d_tgt), _ptr(s), _ptr(t), _ptr(init),
                                               float(max_correspondence_distance), int(max_iteration), _ptr(out),
                                               _ptr(stats[0]) if info else None, _ptr(stats[1]) if info else None,
                                               _ptr(ints[0]) if info else None, _ptr(ints[1]) if info else None,
                                               _ptr(scratch), scratch.numel(), stream))
    if not info:
        return out
    return out, {"fitness": stats[0], "inlier_rmse": stats[1], "iterations": ints[0], "status": ints[1]}


@torch.no_grad()
def information_matrix_packed(src: torch.Tensor, tgt: torch.Tensor, trans: torch.Tensor, src_offsets: Sequence[int],
                              tgt_offsets: Sequence[int], d_src_offsets: Optional[torch.Tensor] = None,
                              d_tgt_offsets: Optional[torch.Tensor] = None, max_correspondence_distance: float = 0.07,
                              status: bool = False):
    """open3d's get_information_matrix_from_point_clouds for B pairs in one call (pdsc_information_matrix_packed).  Pairs and
    offsets as `icp_clouds_packed`; trans [B,4,4] moves each source.  Returns [B,6,6] float64 ([b,5,5] = the correspondences
    kept); with status=True also the [B] int32 status (1: a non-finite coordinate or a target too large for the cell index; the
    matrix is then zero).  Nothing is read back."""
    B, dev, s, t, T, h_src, d_src, h_tgt, d_tgt = _pair_args(src, tgt, src_offsets, tgt_offsets, d_src_offsets, d_tgt_offsets,
                                                             trans, "trans")
    lib, engine, stream = _capi.device_context(dev)
    out = torch.empty(B, 6, 6, dtype=torch.float64, device=dev)
    st = torch.empty(B, dtype=torch.int32, device=dev) if status else None
    scratch = _capi.scratch(lib.pdsc_information_matrix_packed_scratch_bytes(B, h_src, h_tgt), dev)
    with torch.cuda.device(dev):
        _capi.check(lib.pdsc_information_matrix_packed(engine, B, h_src, h_tgt, _ptr(d_src), _ptr(d_tgt), _ptr(s), _ptr(t), _ptr(T),
                                                       float(max_correspondence_distance), _ptr(out), _ptr(st), _ptr(scratch),
                                                       scratch.numel(), stream))
    return (out, st) if status else out


@torch.no_grad()
def multi_scale_icp_packed(clouds: Sequence[torch.Tensor], pairs: Sequence[Tuple[int, int]], inits: torch.Tensor,
                           voxel_sizes: Sequence[float] = (0.05, 0.025, 0.0125), max_iter: Sequence[int] = (50, 30, 14),
                           distance: float = 0.07, status: bool = False):
    """multiway/test_multi_ate.py's `local_refinement` for P pairs (i, j) of `clouds` (device [n,3] tensors) at once: at each
    scale one packed voxel down-sampling of every pair's source and target and one `icp_clouds_packed` call over all pairs
    (max correspondence distance `distance`, starting from the previous scale's result, inits [P,4,4] at the first), then one
    `information_matrix_packed` call at the last scale with r = voxel * 1.4.  Returns (T [P,4,4] float32, info [P,6,6] float64)
    on the device with nothing read back; status=True adds [P] int32, nonzero when a down-sampling, an ICP or the information
    matrix of the pair reported a status."""
    if not pairs:
        raise ValueError("multi_scale_icp_packed needs at least one pair")
    if len(voxel_sizes) != len(max_iter) or not voxel_sizes:
        raise ValueError("voxel_sizes and max_iter must be non-empty and of one length")
    dev = clouds[pairs[0][0]].device
    if dev.type != "cuda":
        raise _capi.PdscError("pointdsc_b200.multiway runs on an H100 only: pass CUDA tensors (there is no CPU fallback)")
    P = len(pairs)
    if tuple(inits.shape) != (P, 4, 4):
        raise ValueError(f"inits must be [{P},4,4], got {tuple(inits.shape)}")
    lib, engine, stream = _capi.device_context(dev)
    # every pair's source, then every pair's target, as 2P clouds of one down-sampling call
    order = [i for i, _ in pairs] + [j for _, j in pairs]
    sizes = [int(clouds[k].shape[0]) for k in order]
    if min(sizes) < 1:
        raise ValueError("every cloud needs at least one point")
    in_off = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    pts = torch.cat([clouds[k].to(torch.float32) for k in order]).contiguous()
    h_in, d_in = _capi.offsets(in_off, None, dev)
    # host bounds of the down-sampled rows: source b ends by in_off[b + 1], target b (rows from the call's output) by in_off[P + b + 1]
    src_bound = in_off[:P + 1]
    tgt_bound = [0] + in_off[P + 1:]
    down = torch.empty(in_off[-1], 3, dtype=torch.float32, device=dev)
    out_off = torch.empty(2 * P + 1, dtype=torch.int32, device=dev)
    vstat = torch.empty(2 * P, dtype=torch.int32, device=dev)
    bad = torch.zeros(P, dtype=torch.int32, device=dev)
    scratch = _capi.scratch(lib.pdsc_voxel_down_sample_packed_scratch_bytes(2 * P, h_in), dev)
    T = inits.to(device=dev, dtype=torch.float32).contiguous()
    for scale, (voxel, iters) in enumerate(zip(voxel_sizes, max_iter)):
        with torch.cuda.device(dev):
            _capi.check(lib.pdsc_voxel_down_sample_packed(engine, 2 * P, h_in, _ptr(d_in), _ptr(pts), float(voxel), _ptr(down),
                                                          _ptr(out_off), _ptr(vstat), _ptr(scratch), scratch.numel(), stream))
        bad |= vstat[:P] | vstat[P:]
        T, st = icp_clouds_packed(down, down, T, src_bound, tgt_bound, d_src_offsets=out_off[:P + 1],
                                  d_tgt_offsets=out_off[P:], max_correspondence_distance=distance, max_iteration=int(iters),
                                  info=True)
        bad |= st["status"]
    info, ist = information_matrix_packed(down, down, T, src_bound, tgt_bound, d_src_offsets=out_off[:P + 1],
                                          d_tgt_offsets=out_off[P:], max_correspondence_distance=float(voxel_sizes[-1]) * 1.4,
                                          status=True)
    bad |= ist
    return (T, info, bad) if status else (T, info)


# ---------------------------------------------------------------------------------------------------------------- pose graph

@dataclass
class PoseGraphEdge:
    source: int
    target: int
    transformation: np.ndarray
    information: np.ndarray
    uncertain: bool = False
    confidence: float = 1.0


@dataclass
class PoseGraph:
    nodes: List[np.ndarray] = field(default_factory=list)        # poses [4,4] float64
    edges: List[PoseGraphEdge] = field(default_factory=list)

    def copy(self) -> "PoseGraph":
        return PoseGraph([p.copy() for p in self.nodes],
                         [PoseGraphEdge(e.source, e.target, e.transformation.copy(), e.information.copy(), e.uncertain, e.confidence)
                          for e in self.edges])


def _colmajor(m: np.ndarray) -> list:
    return [float(x) for x in np.asarray(m, np.float64).flatten(order="F")]


def write_pose_graph(path: str, graph: PoseGraph) -> None:
    """open3d's PoseGraph JSON (write_pose_graph): matrices column-major."""
    doc = {"class_name": "PoseGraph",
           "edges": [{"class_name": "PoseGraphEdge", "confidence": float(e.confidence), "information": _colmajor(e.information),
                      "source_node_id": int(e.source), "target_node_id": int(e.target), "transformation": _colmajor(e.transformation),
                      "uncertain": bool(e.uncertain), "version_major": 1, "version_minor": 0} for e in graph.edges],
           "nodes": [{"class_name": "PoseGraphNode", "pose": _colmajor(p), "version_major": 1, "version_minor": 0}
                     for p in graph.nodes],
           "version_major": 1, "version_minor": 0}
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)


def read_pose_graph(path: str) -> PoseGraph:
    """The inverse of `write_pose_graph` (open3d's read_pose_graph of a .json file)."""
    with open(path) as f:
        doc = json.load(f)
    mat = lambda v, n: np.asarray(v, np.float64).reshape(n, n, order="F")  # noqa: E731
    return PoseGraph([mat(n["pose"], 4) for n in doc["nodes"]],
                     [PoseGraphEdge(int(e["source_node_id"]), int(e["target_node_id"]), mat(e["transformation"], 4),
                                    mat(e["information"], 6), bool(e["uncertain"]), float(e.get("confidence", 1.0)))
                      for e in doc["edges"]])


_GENERATORS = np.zeros((6, 4, 4))
_GENERATORS[0, 1, 2], _GENERATORS[0, 2, 1] = -1.0, 1.0          # rotation about x
_GENERATORS[1, 0, 2], _GENERATORS[1, 2, 0] = 1.0, -1.0          # about y
_GENERATORS[2, 0, 1], _GENERATORS[2, 1, 0] = -1.0, 1.0          # about z
_GENERATORS[3, 0, 3] = _GENERATORS[4, 1, 3] = _GENERATORS[5, 2, 3] = 1.0


def _vec6(E: np.ndarray) -> np.ndarray:
    """[..., 4, 4] -> [..., 6]: (-E[1,2], E[0,2], -E[0,1], E[0,3], E[1,3], E[2,3])."""
    return np.stack([-E[..., 1, 2], E[..., 0, 2], -E[..., 0, 1], E[..., 0, 3], E[..., 1, 3], E[..., 2, 3]], -1)


def _vec6_to_matrix(v: np.ndarray) -> np.ndarray:
    a, b, c = v[0], v[1], v[2]
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    Rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
    M = np.eye(4)
    M[:3, :3] = Rz @ Ry @ Rx
    M[:3, 3] = v[3:]
    return M


def _matrix_to_vec6(M: np.ndarray) -> np.ndarray:
    """The inverse of `_vec6_to_matrix` (open3d's TransformMatrix4dToVector6d): Euler angles (x, y, z) and the translation."""
    R = M[:3, :3]
    sy = np.hypot(R[0, 0], R[1, 0])
    if sy >= 1e-6:
        ang = [np.arctan2(R[2, 1], R[2, 2]), np.arctan2(-R[2, 0], sy), np.arctan2(R[1, 0], R[0, 0])]
    else:
        ang = [np.arctan2(-R[1, 2], R[1, 1]), np.arctan2(-R[2, 0], sy), 0.0]
    return np.concatenate([ang, M[:3, 3]])


class _Edges:
    """The edges of a graph as stacked arrays."""

    def __init__(self, graph: PoseGraph):
        self.s = np.array([e.source for e in graph.edges], np.int64)
        self.t = np.array([e.target for e in graph.edges], np.int64)
        self.X_inv = np.linalg.inv(np.array([e.transformation for e in graph.edges]).reshape(-1, 4, 4))
        self.info = np.array([e.information for e in graph.edges]).reshape(-1, 6, 6)
        self.uncertain = np.array([e.uncertain for e in graph.edges], bool)

    def zeta(self, poses: np.ndarray) -> np.ndarray:
        """[E,6] misalignment vectors."""
        return _vec6(self.X_inv @ np.linalg.inv(poses[self.t]) @ poses[self.s])

    def jacobians(self, poses: np.ndarray):
        A = self.X_inv @ np.linalg.inv(poses[self.t])                       # [E,4,4]
        Js = _vec6(np.einsum("eab,gbc,ecd->egad", A, _GENERATORS, poses[self.s]))    # [E,6 (generator),6 (component)]
        Js = np.swapaxes(Js, 1, 2)                                          # column i = generator i
        return Js, -Js


def _residual(E: _Edges, zeta: np.ndarray, w: float, lp: np.ndarray) -> float:
    quad = np.einsum("ei,eij,ej->e", zeta, E.info, zeta)
    return float(np.sum(lp * quad + w * (np.sqrt(lp) - 1.0) ** 2))


def _update_confidence(E: _Edges, zeta: np.ndarray, w: float, lp: np.ndarray, conf: np.ndarray) -> None:
    quad = np.einsum("ei,eij,ej->e", zeta, E.info, zeta)
    c = (w / (w + quad)) ** 2
    lp[E.uncertain] = c[E.uncertain]
    conf[E.uncertain] = c[E.uncertain]


def _linear_system(E: _Edges, poses: np.ndarray, zeta: np.ndarray, lp: np.ndarray):
    n = len(poses)
    H = np.zeros((6 * n, 6 * n))
    b = np.zeros(6 * n)
    Js, Jt = E.jacobians(poses)
    JsI = np.swapaxes(Js, 1, 2) @ E.info
    JtI = np.swapaxes(Jt, 1, 2) @ E.info
    eI = np.einsum("ei,eij->ej", zeta, E.info)
    for k in range(len(E.s)):
        i, j, l = 6 * E.s[k], 6 * E.t[k], lp[k]
        H[i:i + 6, i:i + 6] += l * JsI[k] @ Js[k]
        H[i:i + 6, j:j + 6] += l * JsI[k] @ Jt[k]
        H[j:j + 6, i:i + 6] += l * JtI[k] @ Js[k]
        H[j:j + 6, j:j + 6] += l * JtI[k] @ Jt[k]
        b[i:i + 6] -= l * eI[k] @ Js[k]
        b[j:j + 6] -= l * eI[k] @ Jt[k]
    return H, b


def optimize_pose_graph(graph: PoseGraph, max_correspondence_distance: float = 0.07, preference_loop_closure: float = 20.0,
                        history: Optional[list] = None) -> PoseGraph:
    """One GlobalOptimizationLevenbergMarquardt::OptimizePoseGraph on a copy of `graph` (no pruning, no reference node): the
    optimised poses and the edges' confidences.  `history`, when given, receives the residual after every accepted step."""
    g = graph.copy()
    if not g.edges:
        return g
    E = _Edges(g)
    poses = np.array(g.nodes)
    w = preference_loop_closure * max_correspondence_distance ** 2 * float(np.mean(E.info[:, 5, 5]))
    lp = np.ones(len(E.s))
    conf = np.array([e.confidence for e in g.edges], np.float64)
    zeta = E.zeta(poses)
    current = _residual(E, zeta, w, lp)
    _update_confidence(E, zeta, w, lp, conf)
    H, b = _linear_system(E, poses, zeta, lp)
    lam = 1e-5 * float(np.max(np.diag(H)))
    ni, rho, eps = 2.0, 0.0, 1e-6
    stop = float(np.max(b)) < eps
    if history is not None:
        history.append(current)
    it = 0
    while not stop:
        lm = 0
        while True:
            delta = np.linalg.solve(H + lam * np.eye(len(b)), b)
            x = np.concatenate([_matrix_to_vec6(p) for p in poses])
            stop = stop or np.linalg.norm(delta) < eps * (np.linalg.norm(x) + eps)
            if not stop:
                new_poses = np.array([_vec6_to_matrix(delta[6 * n:6 * n + 6]) @ poses[n] for n in range(len(poses))])
                new_zeta = E.zeta(new_poses)
                new = _residual(E, new_zeta, w, lp)
                rho = (current - new) / (float(delta @ (lam * delta + b)) + 1e-3)
                if rho > 0:
                    stop = stop or current - new < eps * current
                    alpha = min(1.0 - (2.0 * rho - 1.0) ** 3, 2.0 / 3.0)
                    lam *= max(1.0 / 3.0, alpha)
                    ni = 2.0
                    current = new
                    poses, zeta = new_poses, new_zeta
                    if history is not None:
                        history.append(current)
                    _update_confidence(E, zeta, w, lp, conf)
                    H, b = _linear_system(E, poses, zeta, lp)
                    stop = stop or float(np.max(b)) < eps
                else:
                    lam *= ni
                    ni *= 2.0
            lm += 1
            stop = stop or lm >= 20
            if rho > 0 or stop:
                break
        it += 1
        stop = stop or current < eps or it >= 100
    g.nodes = [p.copy() for p in poses]
    for e, c in zip(g.edges, conf):
        e.confidence = float(c)
    return g


def global_optimization(graph: PoseGraph, max_correspondence_distance: float = 0.07, edge_prune_threshold: float = 0.25,
                        preference_loop_closure: float = 20.0, reference_node: int = 0) -> PoseGraph:
    """open3d 0.9's global_optimization(graph, GlobalOptimizationLevenbergMarquardt(), GlobalOptimizationConvergenceCriteria(),
    GlobalOptimizationOption(max_correspondence_distance, edge_prune_threshold, preference_loop_closure, reference_node)):
    optimise, prune the uncertain edges with confidence <= edge_prune_threshold, optimise again, restore the reference node's
    pose.  Returns the new graph; `graph` is not changed."""
    kw = dict(max_correspondence_distance=max_correspondence_distance, preference_loop_closure=preference_loop_closure)
    g = optimize_pose_graph(graph, **kw)
    g.edges = [e for e in g.edges if not e.uncertain or e.confidence > edge_prune_threshold]
    g = optimize_pose_graph(g, **kw)
    if 0 <= reference_node < len(g.nodes):
        comp = graph.nodes[reference_node] @ np.linalg.inv(g.nodes[reference_node])
        g.nodes = [comp @ p for p in g.nodes]
    return g


def trajectory_ate(gt_poses: Sequence[np.ndarray], est_poses: Sequence[np.ndarray]) -> float:
    """The driver's `align` + RMSE: a Kabsch fit (models/common.py rigid_transform_3d, unit weights, in float64) of the
    ground-truth node positions onto the estimated ones, then sqrt(mean |R g + t - e|^2) in cm."""
    A = np.array([np.asarray(p, np.float64)[:3, 3] for p in gt_poses])
    B = np.array([np.asarray(p, np.float64)[:3, 3] for p in est_poses])
    ca, cb = A.mean(0), B.mean(0)
    U, _, Vt = np.linalg.svd((A - ca).T @ (B - cb))
    D = np.diag([1.0, 1.0, np.linalg.det(Vt.T @ U.T)])
    R = Vt.T @ D @ U.T
    err = np.linalg.norm(A @ R.T + (cb - R @ ca) - B, axis=1) * 100.0
    return float(np.sqrt(np.mean(err ** 2)))
