"""The host-input forward and the two-deep pipeline share one engine: the synchronous call (pdsc_forward_host, model.run with
host tensors) takes a pipeline slot for the length of the call.  It must leave a stream that has a call in flight able to go
on, and a call that fails must leave both slots free.  Needs an H100: `-m gpu`."""
import ctypes as C

import pytest
import torch

from gpu_models import get_model
from pointdsc_b200.model import DEFAULT_PRECISION

pytestmark = pytest.mark.gpu

def host_batch(b, n, seed):
    from pointdsc_b200.synth import make_batch
    mb = make_batch(range(seed, seed + b), n, "3dmatch", 0.4)
    d = {k: mb[k].pin_memory() for k in ("corr_pos", "src_keypts", "tgt_keypts")}
    d["testing"] = True
    return d


def same_result(a, b):
    return torch.equal(a["final_trans"], b["final_trans"]) and torch.equal(a["final_labels"], b["final_labels"])


def test_synchronous_call_beside_a_suspended_stream():
    """model.run with host tensors while a forward_stream generator is suspended with one call in flight: the synchronous
    call (graphed and eager sizes) gives its module result, and the stream then goes on and gives the module results."""
    m = get_model(precision=DEFAULT_PRECISION)
    batches = [host_batch(b, n, 700 + 10 * i) for i, (b, n) in enumerate([(2, 300), (40, 1000), (1, 1000), (3, 400)])]
    between = [host_batch(1, 500, 800), host_batch(40, 1000, 900)]   # B * N on either side of the graph-replay size
    want = [m(d) for d in batches]
    want_between = [m(d) for d in between]
    it = m.forward_stream(iter(batches))
    got = [next(it)]                                   # batch 1 is now in flight
    for d, w in zip(between, want_between):
        assert same_result(m.run(d["corr_pos"], d["src_keypts"], d["tgt_keypts"]), w)
    got += list(it)
    assert len(got) == len(want) and all(same_result(g, w) for g, w in zip(got, want))


def test_failed_host_call_leaves_both_slots_free():
    """pdsc_forward_host refuses N = 20000 (above the largest supported set); afterwards both pipeline slots take a call,
    and the module's host path still gives its result."""
    from pointdsc_b200 import _capi
    m = get_model(precision=DEFAULT_PRECISION)
    lib = m._ensure_engine()
    d = host_batch(2, 300, 950)
    ref = m(d)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: C.c_void_p(t.data_ptr())          # noqa: E731

    n = 20000
    cp, s, t = torch.zeros(1, n, 6).pin_memory(), torch.zeros(1, n, 3).pin_memory(), torch.zeros(1, n, 3).pin_memory()
    tr, lb = torch.empty(1, 4, 4), torch.empty(1, n)
    assert lib.pdsc_forward_host(m._engine, 1, n, P(cp), P(s), P(t), P(tr), P(lb), st) == 7     # PDSC_ERR_UNSUPPORTED
    assert b"exceeds" in lib.pdsc_last_error()

    outs = [(torch.empty(2, 4, 4), torch.empty(2, 300)) for _ in range(2)]
    slots = []
    for o in outs:
        slot = C.c_int32(-1)
        _capi.check(lib.pdsc_forward_host_submit(m._engine, 2, 300, P(d["corr_pos"]), P(d["src_keypts"]), P(d["tgt_keypts"]),
                                                 P(o[0]), P(o[1]), st, C.byref(slot)))
        slots.append(slot.value)
    assert sorted(slots) == [0, 1]
    for sl in slots:
        _capi.check(lib.pdsc_forward_host_wait(m._engine, sl))
    for o in outs:
        assert torch.equal(o[0], ref["final_trans"]) and torch.equal(o[1], ref["final_labels"])
    assert same_result(m.run(d["corr_pos"], d["src_keypts"], d["tgt_keypts"]), ref)
