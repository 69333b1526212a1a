"""Host side of the batch-invariant mode: the module's keyword and setter, the C binding and the driver's flag (no GPU)."""
import ctypes as C
import inspect
import os

from conftest import REPO, load_snapshot


def _model(**kw):
    from pointdsc_b200 import PointDSC
    return PointDSC(num_layers=12, **kw)


def test_keyword_is_keyword_only_and_off_by_default():
    from pointdsc_b200 import PointDSC
    p = inspect.signature(PointDSC.__init__).parameters["batch_invariant"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False
    assert _model().batch_invariant is False
    assert _model(batch_invariant=True).batch_invariant is True


def test_state_dict_is_the_same_in_both_modes():
    off, on = _model(), _model(batch_invariant=True)
    assert list(off.state_dict().keys()) == list(on.state_dict().keys())
    res = on.load_state_dict(load_snapshot("3dmatch"), strict=False)
    assert res.missing_keys == [] and res.unexpected_keys == ["gamma"]


def test_setter_drops_graph_buffers_and_workspaces():
    m = _model()
    m._static[(1, 1000, 0)] = object()
    m._workspaces[0] = object()
    m.set_batch_invariant(True)
    assert m.batch_invariant is True and m._static == {} and m._workspaces == {}
    m.set_batch_invariant(False)
    assert m.batch_invariant is False


def test_binding_declares_the_entry():
    from pointdsc_b200 import _capi
    res, argtypes = _capi.SYMBOLS["pdsc_set_batch_invariant"]
    assert res is C.c_int and argtypes == [C.c_void_p, C.c_int32]
    header = open(os.path.join(REPO, "include", "pointdsc_b200.h")).read()
    assert "int pdsc_set_batch_invariant(pdsc_engine* e, int32_t enable);" in header


def test_evaluate_parses_the_flag():
    import evaluate
    assert evaluate.parse_args(["--synthetic", "4"]).batch_invariant is False
    assert evaluate.parse_args(["--synthetic", "4", "--batch_size", "4", "--batch_invariant"]).batch_invariant is True
