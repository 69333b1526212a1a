"""Device side of the multiway registration (row f7): ICP between two clouds (pdsc_icp_clouds_packed) and information matrices
(pdsc_information_matrix_packed) against float64 (oracle/icp_oracle.py's ICP, tests/multiway_oracle.py's information matrix),
their batch and SM-count invariance, memory and graph contracts and errors, and multiway.py's synthetic scene on the device
against the same pipeline with the float64 restatements on the CPU.

ICP parity is stated as test_gpu_icp.py states it: iterations and fitness exact, rmse within 1e-12 relative and T within 2 float32
ulps, for runs whose every decision clears its threshold by more than 1e-9 (the oracle's margins).  Information parity: the
count [5,5] exact under the same gate, every other entry within 2 gamma_(|C| + 4) sum_c |G_c|^T |G_c| of the float64 value (both
sides sum the same products, in different orders).

One-line kernel mutants and the tests that catch them:
  `<=` for `<` in the radius test            test_information_at_the_radius (targets placed at exactly float32(r^2))
  the source point in G instead of the target test_information_matches_float64 (the off-diagonal blocks)
  the source not moved by T                  test_information_matches_float64, test_two_cloud_icp_matches_oracle
  the target offsets ignored                 test_two_cloud_icp_matches_oracle, test_information_matches_float64 (Ns != Nt)
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from buffer_guards import PATTERNS, assert_same, guarded_input, guarded_output, run_guarded, scratch_buffer
from float64_bounds import gamma64
from gpu_models import get_model, ulps
from multiway_oracle import information_matrix
from oracle import icp_oracle as O

pytestmark = pytest.mark.gpu

MARGIN = 1e-9


def _rigid(rng, deg, shift):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(deg)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K, rng.normal(size=3) * shift
    return T


def _pair(ns, nt, seed):
    """A source of ns rows that overlaps a target of nt rows (a noisy resampling of a surface patch), and a start near truth."""
    rng = np.random.default_rng(seed)
    side = 1.5 * max(1.0, np.sqrt(max(ns, nt) / 200.0))         # ~10 cm between points, so decisions clear their margins
    surf = lambda n: np.c_[rng.uniform(0, side, (n, 2)), np.zeros(n)] + rng.normal(scale=0.004, size=(n, 3))  # noqa: E731
    bump = lambda p: p + np.c_[0 * p[:, :2], 0.3 * np.sin(3 * p[:, 0]) * np.cos(2 * p[:, 1])]  # noqa: E731
    tgt = bump(surf(nt)).astype(np.float32)
    gt = _rigid(rng, 25, 0.5)
    src = ((bump(surf(ns)) - gt[:3, 3]) @ gt[:3, :3]).astype(np.float32)      # gt^-1 applied
    init = (_rigid(rng, 2.0 * 1.5 / side, 0.02) @ gt).astype(np.float32)
    return src, tgt, init


CASES = [(1, 1, 0), (1, 50, 1), (50, 1, 2), (300, 1200, 3), (2000, 700, 4), (100000, 60000, 8)]


def _pack(pairs):
    so = np.cumsum([0] + [len(s) for s, _, _ in pairs]).tolist()
    to = np.cumsum([0] + [len(t) for _, t, _ in pairs]).tolist()
    src = torch.from_numpy(np.concatenate([s for s, _, _ in pairs])).cuda()
    tgt = torch.from_numpy(np.concatenate([t for _, t, _ in pairs])).cuda()
    init = torch.from_numpy(np.stack([i for _, _, i in pairs])).cuda()
    return src, tgt, init, so, to


def _icp(pairs, r=0.07, iters=30):
    from pointdsc_b200.multiway import icp_clouds_packed
    src, tgt, init, so, to = _pack(pairs)
    T, st = icp_clouds_packed(src, tgt, init, so, to, max_correspondence_distance=r, max_iteration=iters, info=True)
    torch.cuda.synchronize()
    return T.cpu().numpy(), {k: v.cpu().numpy() for k, v in st.items()}


def _info(pairs, r=0.07):
    from pointdsc_b200.multiway import information_matrix_packed
    src, tgt, T, so, to = _pack(pairs)
    out, st = information_matrix_packed(src, tgt, T, so, to, max_correspondence_distance=r, status=True)
    torch.cuda.synchronize()
    return out.cpu().numpy(), st.cpu().numpy()


def _info_bound(src, tgt, T, ref):
    """2 gamma_(n + 4) sum_c |G_c|^T |G_c| over the kept correspondences."""
    q = np.abs(np.asarray(tgt, np.float64)[ref["rows"][:, 1]])
    x, y, z = q[:, 0], q[:, 1], q[:, 2]
    zero, one = np.zeros_like(x), np.ones_like(x)
    G = np.stack([np.stack([zero, z, y, one, zero, zero], 1), np.stack([z, zero, x, zero, one, zero], 1),
                  np.stack([y, x, zero, zero, zero, one], 1)], 1)
    return 2.0 * gamma64(len(q) + 4) * np.einsum("cki,ckj->ij", G, G)


# ---------------------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("ns,nt,seed", CASES, ids=[f"ns{a}-nt{b}" for a, b, _ in CASES])
def test_two_cloud_icp_matches_oracle(ns, nt, seed):
    pairs = [_pair(ns, nt, seed), _pair(max(1, nt // 3), max(1, ns // 2), seed + 100)]    # Ns != Nt on both sides of the group
    T, st = _icp(pairs)
    for b, (s, t, i) in enumerate(pairs):
        ref = O.icp(s, t, i, max_correspondence_distance=0.07)
        assert O.margin(ref) > MARGIN, ref["margins"]
        assert int(st["status"][b]) == ref["status"] and int(st["iterations"][b]) == ref["iterations"]
        assert float(st["fitness"][b]) == ref["fitness"]
        assert abs(float(st["inlier_rmse"][b]) - ref["inlier_rmse"]) <= 1e-12 * ref["inlier_rmse"]
        assert ulps(T[b], ref["trans"]).max() <= 2, (T[b], ref["trans"])


def test_icp_packed_is_the_two_cloud_call_with_equal_offsets():
    from pointdsc_b200.icp import icp_refine_packed
    from pointdsc_b200.multiway import icp_clouds_packed
    from pointdsc_b200.synth import make_pair
    sets = [make_pair(s, n, "3dmatch") for s, n in ((0, 1), (1, 700), (2, 3000))]
    off = np.cumsum([0] + [len(p["src_keypts"]) for p in sets]).tolist()
    src = torch.cat([p["src_keypts"] for p in sets]).cuda()
    tgt = torch.cat([p["tgt_keypts"] for p in sets]).cuda()
    init = torch.stack([p["gt_trans"].float() for p in sets]).cuda()
    a, ia = icp_refine_packed(src, tgt, init, off, info=True)
    b, ib = icp_clouds_packed(src, tgt, init, off, off, max_correspondence_distance=0.10, info=True)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    for k in ia:
        assert np.array_equal(ia[k].cpu().numpy(), ib[k].cpu().numpy()), k


@pytest.mark.parametrize("ns,nt,seed", CASES, ids=[f"ns{a}-nt{b}" for a, b, _ in CASES])
def test_information_matches_float64(ns, nt, seed):
    pairs = [_pair(ns, nt, seed), _pair(max(1, nt // 3), max(1, ns // 2), seed + 100)]
    info, st = _info(pairs)
    for b, (s, t, T) in enumerate(pairs):
        ref = information_matrix(s, t, T, 0.07)
        assert min(ref["margins"].values()) > MARGIN, ref["margins"]
        assert int(st[b]) == ref["status"] == 0
        assert info[b, 5, 5] == ref["count"]
        assert np.array_equal(info[b], info[b].T)
        assert (np.abs(info[b] - ref["info"]) <= _info_bound(s, t, T, ref)).all(), np.abs(info[b] - ref["info"]).max()
        if min(len(s), len(t)) >= 50:
            assert ref["count"] > 0


def test_information_at_the_radius():
    """Targets at squared distance exactly float32(r^2) from the moved source are not kept, a hair inside they are."""
    r = 0.0625                                   # r^2 = 2^-8, exact in float32
    src = np.zeros((3, 3), np.float32)
    src[:, 0] = [0.0, 10.0, 20.0]
    tgt = src.copy()
    tgt[0, 1] = r                                # d^2 = r^2: rejected
    tgt[1, 1] = np.nextafter(np.float32(r), np.float32(0))     # just inside: kept
    tgt[2, 1] = 2 * r                            # outside
    info, st = _info([(src, tgt, np.eye(4, dtype=np.float32))], r=r)
    ref = information_matrix(src, tgt, np.eye(4, dtype=np.float32), r)
    assert ref["count"] == 1 and info[0, 5, 5] == 1 and int(st[0]) == 0
    assert np.array_equal(info[0], ref["info"])


def test_status_gives_the_zero_matrix():
    s, t, T = _pair(200, 300, 9)
    bad = s.copy()
    bad[5, 2] = np.inf
    far = t.copy()
    far[0] = [1e6, 0, 0]                          # 2^21 cells or more along x
    info, st = _info([(bad, t, T), (s, far, T), (s, t, T)])
    assert st.tolist()[:2] == [1, 1] and int(st[2]) == 0
    assert not info[:2].any() and info[2, 5, 5] > 0


# ---------------------------------------------------------------------------------------------------------------- invariance
def _group():
    return [_pair(n, m, s) for n, m, s in ((1, 40, 10), (900, 300, 11), (40, 1, 12), (2500, 4000, 13), (7, 7, 14))]


def test_group_alone_and_reversed_are_bit_identical():
    pairs = _group()
    T, st = _icp(pairs)
    info, _ = _info(pairs)
    Tr, _ = _icp(pairs[::-1])
    infor, _ = _info(pairs[::-1])
    for b, p in enumerate(pairs):
        Ta, _ = _icp([p])
        ia, _ = _info([p])
        assert np.array_equal(T[b], Ta[0]) and np.array_equal(T[b], Tr[len(pairs) - 1 - b])
        assert np.array_equal(info[b], ia[0]) and np.array_equal(info[b], infor[len(pairs) - 1 - b])


def test_sm_count_does_not_change_a_bit(tmp_path):
    pairs = _group()
    np.savez(tmp_path / "pairs.npz", *[x for p in pairs for x in p])
    code = f"""
import sys, numpy as np, torch
sys.path.insert(0, {os.path.dirname(os.path.dirname(os.path.abspath(__file__)))!r})
from pointdsc_b200.multiway import icp_clouds_packed, information_matrix_packed
z = np.load(sys.argv[1]); a = [z[f"arr_{{k}}"] for k in range(len(z.files))]
pairs = [a[3 * k:3 * k + 3] for k in range(len(a) // 3)]
so = np.cumsum([0] + [len(p[0]) for p in pairs]).tolist(); to = np.cumsum([0] + [len(p[1]) for p in pairs]).tolist()
s = torch.from_numpy(np.concatenate([p[0] for p in pairs])).cuda(); t = torch.from_numpy(np.concatenate([p[1] for p in pairs])).cuda()
T = torch.from_numpy(np.stack([p[2] for p in pairs])).cuda()
out = icp_clouds_packed(s, t, T, so, to); inf = information_matrix_packed(s, t, T, so, to)
np.savez(sys.argv[2], T=out.cpu().numpy(), info=inf.cpu().numpy())
"""
    res = {}
    for sms in ("", "8"):
        env = dict(os.environ, PDSC_SM_COUNT=sms)
        out = str(tmp_path / f"out{sms}.npz")
        subprocess.run([sys.executable, "-c", code, str(tmp_path / "pairs.npz"), out], env=env, check=True)
        res[sms] = np.load(out)
    assert np.array_equal(res[""]["T"], res["8"]["T"]) and np.array_equal(res[""]["info"], res["8"]["info"])


# ---------------------------------------------------------------------------------------------------------------- contracts
def _raw_info(h_so, h_to, d_so, d_to, src, tgt, T, info, status, scratch, nbytes, r=0.07):
    from pointdsc_b200 import _capi
    lib = _capi.load()
    B = len(h_so) - 1
    return lib.pdsc_information_matrix_packed(_capi.utility_engine(0), B, (C.c_int32 * (B + 1))(*h_so), (C.c_int32 * (B + 1))(*h_to),
                                              C.c_void_p(d_so), C.c_void_p(d_to), C.c_void_p(src), C.c_void_p(tgt), C.c_void_p(T),
                                              float(r), C.c_void_p(info) if info else None, C.c_void_p(status) if status else None,
                                              C.c_void_p(scratch) if scratch else None, nbytes,
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream))


def _raw_icp(h_so, h_to, d_so, d_to, src, tgt, T, outs, scratch, nbytes, r=0.07, iters=30):
    from pointdsc_b200 import _capi
    lib = _capi.load()
    B = len(h_so) - 1
    p = lambda x: C.c_void_p(x) if x else None  # noqa: E731
    return lib.pdsc_icp_clouds_packed(_capi.utility_engine(0), B, (C.c_int32 * (B + 1))(*h_so), (C.c_int32 * (B + 1))(*h_to),
                                      p(d_so), p(d_to), p(src), p(tgt), p(T), float(r), int(iters), *[p(x) for x in outs], p(scratch),
                                      nbytes, C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_guarded_buffers():
    from pointdsc_b200 import _capi
    lib = _capi.load()
    pairs = _group()
    so = np.cumsum([0] + [len(s) for s, _, _ in pairs]).astype(np.int32)
    to = np.cumsum([0] + [len(t) for _, t, _ in pairs]).astype(np.int32)
    B = len(pairs)
    dev = torch.device("cuda")
    ins = {"src": guarded_input(np.concatenate([s for s, _, _ in pairs]), dev), "tgt": guarded_input(np.concatenate([t for _, t, _ in pairs]), dev),
           "T": guarded_input(np.stack([i for _, _, i in pairs]), dev), "so": guarded_input(so, dev), "to": guarded_input(to, dev)}
    h_so, h_to = so.tolist(), to.tolist()
    need_i = int(lib.pdsc_information_matrix_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*h_so), (C.c_int32 * (B + 1))(*h_to)))
    need_c = int(lib.pdsc_icp_clouds_packed_scratch_bytes(B, (C.c_int32 * (B + 1))(*h_so), (C.c_int32 * (B + 1))(*h_to)))
    assert need_i > 0 and need_c > 0
    refs = {}
    for pat in PATTERNS:
        outs = {"info": guarded_output(B * 288, 8, dev, pat), "status": guarded_output(B * 4, 4, dev, pat),
                "trans": guarded_output(B * 64, 4, dev, pat), "fitness": guarded_output(B * 8, 8, dev, pat),
                "rmse": guarded_output(B * 8, 8, dev, pat), "its": guarded_output(B * 4, 4, dev, pat),
                "icp_status": guarded_output(B * 4, 4, dev, pat)}
        sc = scratch_buffer(max(need_i, need_c), 8, pat)
        a = run_guarded(("info", pat), {k: outs[k] for k in ("info", "status")}, sc, ins,
                        lambda: _raw_info(h_so, h_to, ins["so"].ptr, ins["to"].ptr, ins["src"].ptr, ins["tgt"].ptr, ins["T"].ptr,
                                          outs["info"].ptr, outs["status"].ptr, sc.ptr, need_i))
        keys = ("trans", "fitness", "rmse", "its", "icp_status")
        b = run_guarded(("icp", pat), {k: outs[k] for k in keys}, sc, ins,
                        lambda: _raw_icp(h_so, h_to, ins["so"].ptr, ins["to"].ptr, ins["src"].ptr, ins["tgt"].ptr, ins["T"].ptr,
                                         [outs[k].ptr for k in keys], sc.ptr, need_c))
        got = dict(a, **b)
        if refs:
            assert_same(refs, got, (pat,))
        else:
            refs = got


def test_graph_replay_is_bit_identical():
    from pointdsc_b200.multiway import information_matrix_packed, multi_scale_icp_packed
    pairs = _group()
    src, tgt, T, so, to = _pack(pairs)
    d_so = torch.tensor(so, dtype=torch.int32, device="cuda")
    d_to = torch.tensor(to, dtype=torch.int32, device="cuda")
    clouds = [torch.from_numpy(x).cuda() for p in pairs for x in p[:2]]
    idx = [(2 * k, 2 * k + 1) for k in range(len(pairs))]
    eager = information_matrix_packed(src, tgt, T, so, to, d_so, d_to)
    msi = multi_scale_icp_packed(clouds, idx, T)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        information_matrix_packed(src, tgt, T, so, to, d_so, d_to)       # warm-up outside the capture
        with torch.cuda.graph(g, stream=s):
            graphed = information_matrix_packed(src, tgt, T, so, to, d_so, d_to)
    torch.cuda.current_stream().wait_stream(s)
    graphed.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager, graphed)
    again = multi_scale_icp_packed(clouds, idx, T)
    assert torch.equal(msi[0], again[0]) and torch.equal(msi[1], again[1])


def test_errors():
    from pointdsc_b200 import _capi
    from pointdsc_b200.multiway import icp_clouds_packed, information_matrix_packed
    lib = _capi.load()
    pairs = _group()[:3]
    src, tgt, T, so, to = _pack(pairs)
    d_so = torch.tensor(so, dtype=torch.int32, device="cuda")
    d_to = torch.tensor(to, dtype=torch.int32, device="cuda")
    B = len(pairs)
    H = lambda v: (C.c_int32 * len(v))(*v)  # noqa: E731
    need = int(lib.pdsc_information_matrix_packed_scratch_bytes(B, H(so), H(to)))
    sc = torch.empty(need + 16, dtype=torch.uint8, device="cuda")
    info = torch.empty(B, 6, 6, dtype=torch.float64, device="cuda")
    args = (d_so.data_ptr(), d_to.data_ptr(), src.data_ptr(), tgt.data_ptr(), T.data_ptr(), info.data_ptr(), None)
    assert _raw_info(so, to, *args, sc.data_ptr(), need) == 0
    bad_to = [0, to[1], to[1], to[3]]
    assert _raw_info(so, bad_to, *args, sc.data_ptr(), need) == 3
    assert "target" in lib.pdsc_last_error().decode()
    assert _raw_info([1] + so[1:], to, *args, sc.data_ptr(), need) == 3
    assert lib.pdsc_information_matrix_packed_scratch_bytes(B, H(so), H(bad_to)) == 0
    assert lib.pdsc_icp_clouds_packed_scratch_bytes(B, H(bad_to), H(to)) == 0
    for r in (0.0, -1.0, float("nan"), float("inf")):
        assert _raw_info(so, to, *args, sc.data_ptr(), need, r=r) == 1
    assert _raw_info(so, to, *args[:5], None, None, sc.data_ptr(), need) == 1
    assert _raw_info(so, to, *args, sc.data_ptr(), need - 1) == 5
    assert _raw_info(so, to, *args, sc.data_ptr() + 4, need) == 5
    need_c = int(lib.pdsc_icp_clouds_packed_scratch_bytes(B, H(so), H(to)))
    sc_c = torch.empty(need_c, dtype=torch.uint8, device="cuda")
    out = torch.empty(B, 4, 4, device="cuda")
    base = (d_so.data_ptr(), d_to.data_ptr(), src.data_ptr(), tgt.data_ptr(), T.data_ptr())
    outs = [out.data_ptr(), None, None, None, None]
    assert _raw_icp(so, to, *base, outs, sc_c.data_ptr(), need_c) == 0
    assert _raw_icp(so, to, *base, outs, sc_c.data_ptr(), need_c, iters=0) == 1
    assert _raw_icp(so, bad_to, *base, outs, sc_c.data_ptr(), need_c) == 3
    assert _raw_icp(so, to, *base, outs, sc_c.data_ptr(), need_c - 1) == 5
    assert "pdsc_icp_clouds_packed" in lib.pdsc_last_error().decode()
    with pytest.raises(ValueError):
        icp_clouds_packed(src, tgt, T, so, to[:-1])
    with pytest.raises(ValueError):
        information_matrix_packed(src, tgt[:-1], T, so, to)
    with pytest.raises(_capi.PdscError):
        information_matrix_packed(src.cpu(), tgt.cpu(), T.cpu(), so, to)


# ---------------------------------------------------------------------------------------------------------------- the driver
def _oracle_ops(monkeypatch):
    """multi_scale_icp_packed and information_matrix_packed restated on the CPU with the float64 oracles."""
    from oracle import fpfh_oracle as F
    from pointdsc_b200 import multiway as mw

    def msi(clouds, pairs, inits, voxel_sizes=(0.05, 0.025, 0.0125), max_iter=(50, 30, 14), distance=0.07, status=False):
        T_out, I_out = [], []
        for (i, j), T in zip(pairs, inits.cpu().numpy()):
            a, b = clouds[i].cpu().numpy(), clouds[j].cpu().numpy()
            for v, it in zip(voxel_sizes, max_iter):
                s = F.voxel_down_sample(a, v)[0].astype(np.float32)
                t = F.voxel_down_sample(b, v)[0].astype(np.float32)
                T = O.icp(s, t, T, max_correspondence_distance=distance, max_iteration=it)["trans"]
            T_out.append(T)
            I_out.append(information_matrix(s, t, T, voxel_sizes[-1] * 1.4)["info"])
        return torch.from_numpy(np.stack(T_out)), torch.from_numpy(np.stack(I_out))

    def info(src, tgt, trans, so, to, d_src_offsets=None, d_tgt_offsets=None, max_correspondence_distance=0.07, status=False):
        s, t, T = src.cpu().numpy(), tgt.cpu().numpy(), trans.cpu().numpy()
        return torch.from_numpy(np.stack([information_matrix(s[so[b]:so[b + 1]], t[to[b]:to[b + 1]], T[b],
                                                               max_correspondence_distance)["info"] for b in range(len(so) - 1)]))

    monkeypatch.setattr(mw, "multi_scale_icp_packed", msi)
    monkeypatch.setattr(mw, "information_matrix_packed", info)


def test_synthetic_scene_device_against_float64(monkeypatch, tmp_path):
    """multiway.py on a synthetic scene of 6 fragments: the device run and the same run with the ICP, down-sampling and
    information matrices of the float64 oracles keep the same loop closures, prune the same edges, and end within 1 mm / 1e-3 of
    each other in every pose entry (ICP's T agrees to float32 rounding; the optimisation is the same host code on both)."""
    import multiway as driver
    from pointdsc_b200 import multiway as mw
    model = get_model("3dmatch", "fp32")
    data = driver.synthetic_scene(6, 0, "cuda")
    quiet = lambda *_: None  # noqa: E731
    g_dev, ate_dev = driver.run_scene(model, data, str(tmp_path / "dev"), batch_size=4, log=quiet)
    with monkeypatch.context() as m:
        _oracle_ops(m)
        g_cpu, ate_cpu = driver.run_scene(model, data, str(tmp_path / "cpu"), batch_size=4, log=quiet)
    for k in ("_0", "_1", "_2"):
        a, b = mw.read_pose_graph(str(tmp_path / f"dev{k}.json")), mw.read_pose_graph(str(tmp_path / f"cpu{k}.json"))
        assert [(e.source, e.target, e.uncertain) for e in a.edges] == [(e.source, e.target, e.uncertain) for e in b.edges], k
        assert max(np.abs(x - y).max() for x, y in zip(a.nodes, b.nodes)) < 1e-3, k
    assert abs(ate_dev - ate_cpu) < 0.1
    assert ate_dev < 10.0                          # cm: the synthetic trajectory is recovered
