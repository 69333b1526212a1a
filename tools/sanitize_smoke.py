#!/usr/bin/env python
"""Developer tool: a small pass through every C-ABI entry for compute-sanitizer:
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py"""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from pointdsc_b200 import PointDSC
from pointdsc_b200.frontend import match, match_many
from pointdsc_b200.metrics import eval_stats, eval_stats_packed
from pointdsc_b200.spectral import leading_eigenvector
for k, n, b, inv in ((40, 300, 3, False), (80, 257, 2, False), (40, 1000, 2, True)):   # the last: batch-invariant key split
    m = PointDSC(num_layers=12, k=k, batch_invariant=inv, **bench.CTOR["3dmatch"]); m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False); m = m.cuda().eval()
    h = bench.make_inputs(n, b, "3dmatch", 0)
    d = [h[x].cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")]
    out = m.run(*d, taps=["best"])                      # eager
    dbg = m.run(*d, taps=["layer_debug"], layer_tap=3)   # the debug tap un-blocks feat1
    out2 = m.run(*d)                                    # graph path (capture + replay)
    out2 = m.run(*d)
    ev = m({"corr_pos": d[0], "src_keypts": d[1], "tgt_keypts": d[2]})
    st = eval_stats(out["final_trans"], h["gt_trans"].cuda(), d[1], d[2], out["final_labels"], h["gt_labels"].cuda())
    v, it = leading_eigenvector(ev["M"], 10, True)
    host = m.run(h["corr_pos"], h["src_keypts"], h["tgt_keypts"])
    hd = {"corr_pos": h["corr_pos"].pin_memory(), "src_keypts": h["src_keypts"].pin_memory(), "tgt_keypts": h["tgt_keypts"].pin_memory(),
          "testing": True}
    streamed = list(m.forward_stream(hd for _ in range(3)))      # pdsc_forward_host_submit / _wait, two calls in flight
    assert all(torch.equal(o["final_trans"], host["final_trans"]) for o in streamed)
    mixed = [bench.make_inputs(nn, 1, "3dmatch", 0) for nn in (n, 41, 7, 130)]   # pdsc_forward_packed, sets of four sizes
    many = m.forward_many([{**{x: q[x].cuda() for x in ("corr_pos", "src_keypts", "tgt_keypts")}, "testing": True} for q in mixed])
    assert [tuple(o["final_labels"].shape) for o in many] == [(1, n), (1, 41), (1, 7), (1, 130)]
for prec in ("bf16x3", "bf16"):   # the bf16 instantiations of every chain mode (PCQ, Q, KV, MSGPC, MSG), split on and off
    m = PointDSC(num_layers=12, k=40, precision=prec, **bench.CTOR["3dmatch"]); m.load_state_dict(bench.load_snapshot("3dmatch"), strict=False); m = m.cuda().eval()
    m.run(*d, taps=["layer_features", "layer_debug"], layer_tap=5)   # layer 5's MSGPC also writes feat for the tap
g = torch.Generator().manual_seed(0)
for dt in (torch.float32, torch.float64):
    sd = torch.nn.functional.normalize(torch.randn(301, 33, generator=g, dtype=dt), dim=1).cuda()
    td = torch.nn.functional.normalize(torch.randn(277, 33, generator=g, dtype=dt), dim=1).cuda()
    for mutual in (False, True):
        r = match(sd, td, torch.rand(301, 3).cuda(), torch.rand(277, 3).cuda(), use_mutual=mutual)
        pk = match_many([(sd, td, torch.rand(301, 3).cuda(), torch.rand(277, 3).cuda()), (sd[:1], td[:70], torch.rand(1, 3).cuda(),
                         torch.rand(70, 3).cuda()), (sd[:130], td[:1], torch.rand(130, 3).cuda(), torch.rand(1, 3).cuda())],
                        use_mutual=mutual)                       # pdsc_match_packed, pairs of three sizes
        off = pk["offsets"]
        sp = eval_stats_packed(torch.eye(4).expand(3, 4, 4).cuda(), torch.eye(4).expand(3, 4, 4).cuda(), pk["src_keypts"],
                               pk["tgt_keypts"], pk["corr_pos"][:, 0], pk["corr_pos"][:, 1], off, d_offsets=pk["d_offsets"])
from pointdsc_b200 import descriptors as D
from pointdsc_b200.synth_scene import scene
kp, feat = D.fpfh_descriptors(torch.from_numpy(scene(4000, seed=0)).cuda(), 0.15)
kp_many, feat_many, _, _ = D.fpfh_descriptors_many([torch.from_numpy(scene(nn, seed=nn)).cuda() for nn in (4000, 1, 700)], 0.15)  # the packed calls
from pointdsc_b200.icp import icp_refine, icp_refine_packed
ic = icp_refine(h["src_keypts"].cuda(), h["tgt_keypts"].cuda(), out["final_trans"])
ip, ii = icp_refine_packed(pk["src_keypts"], pk["tgt_keypts"], torch.eye(4).expand(3, 4, 4).cuda(), off, d_offsets=pk["d_offsets"],
                           info=True)                    # pdsc_icp_packed, sets of three sizes
from pointdsc_b200.spectral import spectral_matching_packed
smt, sml = spectral_matching_packed(pk["corr_pos"], pk["src_keypts"], pk["tgt_keypts"], off, d_offsets=pk["d_offsets"])  # sets of three sizes
torch.cuda.synchronize()
print("sanitize_smoke ok", float(st.sum()), int(it.sum()), r["corr"].shape, tuple(feat.shape))
