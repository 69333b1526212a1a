"""Host-side logic of evaluate.py --solver RANSAC: after the forward, RANSAC replaces the transform and the labels, then --use_icp
refines the transform, then the statistics run on RANSAC's labels; RANSAC and ICP sit inside the model-time events; once per pair
(bs = 1 and the forward_many fallback) or once per packed group.  Without the flag RANSAC never runs."""
import numpy as np
import pytest
import torch

import evaluate
from fakes import _PackedModel, _fake_packed, _fake_pipeline

R_3DMATCH = 0.10


def _fakes(monkeypatch, log, seen):
    import pointdsc_b200.icp as icp
    import pointdsc_b200.metrics as me
    import pointdsc_b200.ransac as ra

    def ransac_refine(src, tgt, pred_labels, max_correspondence_distance=0.10, max_iteration=5000, seed=51):
        log.append("ransac_refine")
        assert max_correspondence_distance == R_3DMATCH and pred_labels.shape == src.shape[:2]
        return torch.eye(4)[None] * 3.0, torch.full_like(pred_labels, 7.0)

    def ransac_packed(src, tgt, labels, offsets, d_offsets=None, max_correspondence_distance=0.10, max_iteration=5000, seed=51,
                      info=False, hypotheses=False):
        log.append("ransac_packed")
        assert d_offsets is not None and max_correspondence_distance == R_3DMATCH and labels.shape == (offsets[-1],)
        return torch.eye(4).expand(len(offsets) - 1, 4, 4) * 3.0, torch.full_like(labels, 7.0)

    def icp_refine(src, tgt, trans, max_correspondence_distance=0.10):
        log.append("icp_refine")
        return trans * 2.0

    def icp_refine_packed(src, tgt, trans, offsets, d_offsets=None, max_correspondence_distance=0.10, max_iteration=30, info=False):
        log.append("icp_refine_packed")
        return trans * 2.0

    def eval_stats(trans, gt, src, tgt, labels, gt_labels, re_thre, te_thre):
        log.append("eval_stats")
        seen.append(float(labels.reshape(-1)[0]))
        return torch.full((1, 10), float(trans[0, 0, 0]))

    packed_stats = me.eval_stats_packed

    def eval_stats_packed(trans, gt, src, tgt, labels, *args, **kw):
        out = packed_stats(trans, gt, src, tgt, labels, *args, **kw)
        seen.append(float(labels[0]))
        out[:, 1] = trans[:, 0, 0]
        return out

    monkeypatch.setattr(ra, "ransac_refine", ransac_refine)
    monkeypatch.setattr(ra, "ransac_packed", ransac_packed)
    monkeypatch.setattr(icp, "icp_refine", icp_refine)
    monkeypatch.setattr(icp, "icp_refine_packed", icp_refine_packed)
    monkeypatch.setattr(me, "eval_stats", eval_stats)
    monkeypatch.setattr(me, "eval_stats_packed", eval_stats_packed)


class _LoggedModel(_PackedModel):
    def __call__(self, data):
        self.log.append("forward")
        return super().__call__(data)


class _ManyModel:
    """A model with the mixed-size interface only: evaluate groups it pair by pair."""

    def __init__(self, log):
        self.log = log

    def forward_many(self, datas):
        self.log.append("forward_many")
        return [{"final_trans": torch.eye(4)[None], "final_labels": torch.ones(1, d["src_keypts"].shape[1])} for d in datas]


def _run(monkeypatch, model_cls, batch_size, solver, use_icp):
    log, seen, events = [], [], []
    _fake_pipeline(monkeypatch)
    _fake_packed(monkeypatch, log)
    _fakes(monkeypatch, log, seen)
    record = evaluate.torch.cuda.Event.record

    def logged_record(self):
        events.append(len(log))
        record(self)
    monkeypatch.setattr(evaluate.torch.cuda.Event, "record", logged_record)
    cfg = {"inlier_threshold": R_3DMATCH, "re_thre": 15.0, "te_thre": 30.0}
    pairs = [(0, (None, n), (None, n), np.eye(4)) for n in (30, 40, 50)]
    out = evaluate.evaluate(model_cls(log), pairs, cfg, device="cpu", batch_size=batch_size, use_icp=use_icp, solver=solver)
    return log, seen, events, out


@pytest.mark.parametrize("use_icp", [False, True])
@pytest.mark.parametrize("solver", ["SVD", "RANSAC"])
def test_per_pair_order_events_and_labels(monkeypatch, solver, use_icp):
    log, seen, events, out = _run(monkeypatch, _LoggedModel, 1, solver, use_icp)
    step = ["forward"] + (["ransac_refine"] if solver == "RANSAC" else []) + (["icp_refine"] if use_icp else []) + ["eval_stats"]
    assert log == step * 3
    for p in range(3):                                           # the events enclose the forward, RANSAC and ICP, not the statistics
        assert log[events[2 * p]:events[2 * p + 1]] == step[:-1]
    assert seen == [7.0 if solver == "RANSAC" else 1.0] * 3      # the statistics get RANSAC's labels
    assert list(out[:, 0]) == [(3.0 if solver == "RANSAC" else 1.0) * (2.0 if use_icp else 1.0)] * 3


@pytest.mark.parametrize("use_icp", [False, True])
@pytest.mark.parametrize("solver", ["SVD", "RANSAC"])
def test_packed_order_events_and_labels(monkeypatch, solver, use_icp):
    log, seen, events, out = _run(monkeypatch, _PackedModel, 2, solver, use_icp)
    step = ["match_many", "forward_packed"] + (["ransac_packed"] if solver == "RANSAC" else []) + \
        (["icp_refine_packed"] if use_icp else []) + ["eval_stats_packed"]
    assert log == step * 2
    for g in range(2):
        assert log[events[2 * g]:events[2 * g + 1]] == step[1:-1]
    assert seen == [7.0 if solver == "RANSAC" else 1.0] * 2
    assert list(out[:, 1]) == [(3.0 if solver == "RANSAC" else 1.0) * (2.0 if use_icp else 1.0)] * 3


@pytest.mark.parametrize("use_icp", [False, True])
def test_forward_many_fallback_runs_ransac_per_pair(monkeypatch, use_icp):
    log, seen, events, out = _run(monkeypatch, _ManyModel, 2, "RANSAC", use_icp)
    per = ["ransac_refine"] + (["icp_refine"] if use_icp else [])
    assert log == ["forward_many"] + per * 2 + ["eval_stats"] * 2 + ["forward_many"] + per + ["eval_stats"]
    assert log[events[0]:events[1]] == ["forward_many"] + per * 2
    assert seen == [7.0] * 3


def test_solver_flag():
    assert evaluate.parse_args([]).solver == "SVD"
    assert evaluate.parse_args(["--solver", "RANSAC"]).solver == "RANSAC"
    assert evaluate.parse_args(["--solver", "RANSAC", "--use_icp"]).use_icp is True
    with pytest.raises(SystemExit):
        evaluate.parse_args(["--solver", "ransac"])
    with pytest.raises(ValueError):
        evaluate.evaluate(None, [], {}, solver="LM")
