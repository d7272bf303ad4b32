"""The embedding lookups of the layer API -- EmbeddingCollection.forward (ops.EmbedFM) and ops.FnnInputFn -- in every
gradient mode: dense .grad buffers, fused sparse SGD (sparse_lr) and RowSparseAdam.

Launch plans: a proxy in front of the library records the name of every dr_* call.  Each case pins the calls of the
forward, of the backward and, under RowSparseAdam, of step(), and which of weight.grad, linear.grad and bias.grad is
None (DESIGN.md 4k).  The cases cover the fused (D 16), split (D 32) and first-order-free (D 16) collections, plain
lookups and lookups with one bag slot, and the outputs a model uses: stack and logit, the stack alone, and xDeepFM's
linear unit (second_order=False).

Bags of one: when every bag of a slot holds exactly that example's single-valued id, the bag path must give what the
plain lookup gives -- stack, logit, table gradients and the parameters after one step, in all three modes.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
ROWS = [13, 9, 21]
B = 64
BAG_SLOT = 1
COLLECTIONS = {"fused16": dict(dim=16, layout="fused"), "split32": dict(dim=32, layout="split"),
               "nolin16": dict(dim=16, with_linear=False)}


class _Recorder:
    """Stands in for the loaded library: records (name, args) of every dr_* call and forwards it."""

    def __init__(self, lib):
        self._lib = lib
        self.calls = []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("dr_"):
            return fn

        def call(*args):
            self.calls.append((name, args))
            return fn(*args)
        return call

    def take(self):
        torch.cuda.synchronize()
        calls, self.calls = self.calls, []
        return calls


@pytest.fixture
def recorder(monkeypatch):
    from deep_recommenders_b200 import _lib
    rec = _Recorder(_lib.load())
    monkeypatch.setattr(_lib, "_lib", rec)
    return rec


def _collection(kind, mode):
    from deep_recommenders_b200.embedding import EmbeddingCollection
    from deep_recommenders_b200.optimizers import RowSparseAdam
    coll = EmbeddingCollection(ROWS, device=DEV, seed=0, sparse_lr=0.05 if mode == "sgd" else None,
                               **COLLECTIONS[kind])
    if coll.with_linear:
        g = torch.Generator(device=DEV).manual_seed(1)
        with torch.no_grad():
            coll.lin_view().copy_(torch.randn(coll.total_rows, device=DEV, generator=g) / 4)
            coll.bias.fill_(0.25)
    opt = RowSparseAdam(coll, 0.01) if mode == "adam" else None
    return coll, opt


def _ids(seed=2):
    """[B, S] ids with duplicates and pruned (-1, >= rows) entries."""
    rng = np.random.default_rng(seed)
    ids = np.stack([rng.integers(-1, n + 2, B) for n in ROWS], axis=1)
    return torch.from_numpy(ids).to(DEV)


def _bags(seed=3):
    """Slot BAG_SLOT as a bag of 0..3 ids per example: empty bags, duplicate and pruned members."""
    rng = np.random.default_rng(seed)
    n = ROWS[BAG_SLOT]
    per = [list(rng.integers(-1, n + 2, int(rng.integers(0, 4)))) for _ in range(B)]
    per[0], per[1] = [], [0, 0, n + 1]
    flat = torch.tensor([v for p in per for v in p], dtype=torch.int64, device=DEV)
    splits = torch.tensor(np.cumsum([0] + [len(p) for p in per]), dtype=torch.int64, device=DEV)
    return {BAG_SLOT: (flat, splits)}


def _bags_of_one(ids):
    """Every bag of slot BAG_SLOT holds that example's id of ids, the plain lookup's."""
    return {BAG_SLOT: (ids[:, BAG_SLOT].contiguous(), torch.arange(B + 1, dtype=torch.int64, device=DEV))}


def _upstream(shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, device=DEV, generator=g)


def _grad_state(coll):
    """Which of weight.grad, linear.grad and bias.grad is None: 'N' None, 'T' a tensor, '-' no such parameter."""
    return "".join("-" if p is None else ("N" if p.grad is None else "T") for p in (coll.weight, coll.linear, coll.bias))


def _run_embed(coll, opt, rec, use, bags):
    """One forward, backward and (under RowSparseAdam) step() of the collection.  Returns the launch plan and the
    tensors: stack, logit, the gradients and the parameters after the step."""
    ids = _ids()
    want_logit, second_order = use != "stack", use != "linear"
    stack, logit = coll(ids, want_logit=want_logit, bags=bags, second_order=second_order)
    fwd = rec.take()
    loss = (stack * _upstream(stack.shape, 4)).sum()
    if want_logit:
        loss = loss + (logit * _upstream(logit.shape, 5)).sum()
    loss.backward()
    bwd = rec.take()
    if opt is not None:
        opt.step()
    step = rec.take()
    out = {"stack": stack, "logit": logit}
    for name in ("weight", "linear", "bias"):
        p = getattr(coll, name)
        if p is not None:
            out[name] = p
            out["d" + name] = p.grad
    return (fwd, bwd, step, _grad_state(coll)), out


def _run_fnn(coll, opt, rec, bags):
    from deep_recommenders_b200 import ops
    ids = _ids()
    bias = torch.full((1,), 0.5, device=DEV)
    x = ops.FnnInputFn.apply(ids, coll.weight, coll.linear, bias, coll, bags)
    fwd = rec.take()
    (x * _upstream(x.shape, 6)).sum().backward()
    bwd = rec.take()
    if opt is not None:
        opt.step()
    step = rec.take()
    out = {"x": x, "weight": coll.weight, "dweight": coll.weight.grad}
    if coll.linear is not None:
        out.update(linear=coll.linear, dlinear=coll.linear.grad)
    return (fwd, bwd, step, _grad_state(coll)), out


def _names(calls):
    return [name for name, _ in calls]


MODES = ("dense", "sgd", "adam")
EMBED_CASES = [(kind, lookup, use, mode) for mode in MODES for kind in COLLECTIONS for lookup in ("plain", "bag")
               for use in ("both", "stack", "linear")
               if not (kind == "nolin16" and use != "stack") and not (lookup == "bag" and use == "linear")]
FNN_CASES = [(kind, lookup, mode) for mode in MODES for kind in ("fused16", "split32") for lookup in ("plain", "bag")]

CATCH_UP, FM_FWD, FM_BWD, BAG_FWD, BAG_BWD = ("dr_embed_adam_catch_up", "dr_embed_fm_fwd", "dr_embed_fm_bwd",
                                               "dr_embed_bag_fwd", "dr_embed_bag_bwd")
COLSUM, ADVANCE, COUNT, FM_ADAM, ROWS_ADAM = ("dr_act_bwd_colsum", "dr_adam_advance_hist", "dr_embed_adam_count",
                                              "dr_embed_fm_bwd_adam_tf", "dr_embed_adam_rows_tf")
FNN_FWD, FNN_BWD = "dr_fnn_input_fwd", "dr_fnn_input_bwd"

# (forward, backward, step(), grad state of weight / linear / bias) per case; the no_grad cases: the forward only
PLANS = {
    ("embed", "fused16", "plain", "both", "dense"): ([FM_FWD], [FM_BWD], [], "T-T"),
    ("embed", "fused16", "plain", "stack", "dense"): ([FM_FWD], [FM_BWD], [], "T-N"),
    ("embed", "fused16", "plain", "linear", "dense"): ([FM_FWD], [FM_BWD], [], "T-T"),
    ("embed", "fused16", "bag", "both", "dense"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "T-T"),
    ("embed", "fused16", "bag", "stack", "dense"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "T-T"),
    ("embed", "split32", "plain", "both", "dense"): ([FM_FWD], [FM_BWD], [], "TTT"),
    ("embed", "split32", "plain", "stack", "dense"): ([FM_FWD], [FM_BWD], [], "TNN"),
    ("embed", "split32", "plain", "linear", "dense"): ([FM_FWD], [FM_BWD], [], "TTT"),
    ("embed", "split32", "bag", "both", "dense"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "TTT"),
    ("embed", "split32", "bag", "stack", "dense"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "TTT"),
    ("embed", "nolin16", "plain", "stack", "dense"): ([FM_FWD], [FM_BWD], [], "T--"),
    ("embed", "nolin16", "bag", "stack", "dense"): ([BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD], [], "T--"),
    ("embed", "fused16", "plain", "both", "sgd"): ([FM_FWD], [FM_BWD], [], "N-N"),
    ("embed", "fused16", "plain", "stack", "sgd"): ([FM_FWD], [FM_BWD], [], "N-N"),
    ("embed", "fused16", "plain", "linear", "sgd"): ([FM_FWD], [FM_BWD], [], "N-N"),
    ("embed", "fused16", "bag", "both", "sgd"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "N-N"),
    ("embed", "fused16", "bag", "stack", "sgd"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "N-N"),
    ("embed", "split32", "plain", "both", "sgd"): ([FM_FWD], [FM_BWD], [], "NNN"),
    ("embed", "split32", "plain", "stack", "sgd"): ([FM_FWD], [FM_BWD], [], "NNN"),
    ("embed", "split32", "plain", "linear", "sgd"): ([FM_FWD], [FM_BWD], [], "NNN"),
    ("embed", "split32", "bag", "both", "sgd"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "NNN"),
    ("embed", "split32", "bag", "stack", "sgd"): ([BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD, BAG_BWD], [], "NNN"),
    ("embed", "nolin16", "plain", "stack", "sgd"): ([FM_FWD], [FM_BWD], [], "N--"),
    ("embed", "nolin16", "bag", "stack", "sgd"): ([BAG_FWD, FM_FWD], [FM_BWD, BAG_BWD], [], "N--"),
    ("embed", "fused16", "plain", "both", "adam"): ([CATCH_UP, FM_FWD], [COLSUM], [ADVANCE, COUNT, FM_ADAM], "N-T"),
    ("embed", "fused16", "plain", "stack", "adam"): ([CATCH_UP, FM_FWD], [], [ADVANCE, COUNT, ROWS_ADAM], "N-N"),
    ("embed", "fused16", "plain", "linear", "adam"): ([CATCH_UP, FM_FWD], [COLSUM], [ADVANCE, COUNT, ROWS_ADAM], "N-T"),
    ("embed", "fused16", "bag", "both", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "N-T"),
    ("embed", "fused16", "bag", "stack", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "N-T"),
    ("embed", "split32", "plain", "both", "adam"): ([CATCH_UP, FM_FWD], [COLSUM], [ADVANCE, COUNT, FM_ADAM], "NNT"),
    ("embed", "split32", "plain", "stack", "adam"): ([CATCH_UP, FM_FWD], [], [ADVANCE, COUNT, ROWS_ADAM], "NNN"),
    ("embed", "split32", "plain", "linear", "adam"): ([CATCH_UP, FM_FWD], [COLSUM], [ADVANCE, COUNT, ROWS_ADAM], "NNT"),
    ("embed", "split32", "bag", "both", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "NNT"),
    ("embed", "split32", "bag", "stack", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FM_FWD], [FM_BWD], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "NNT"),
    ("embed", "nolin16", "plain", "stack", "adam"): ([CATCH_UP, FM_FWD], [], [ADVANCE, COUNT, ROWS_ADAM], "N--"),
    ("embed", "nolin16", "bag", "stack", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, FM_FWD], [], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "N--"),
    ("no_grad", "plain"): [CATCH_UP, FM_FWD],
    ("no_grad", "bag"): [CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FM_FWD],
    ("fnn", "fused16", "plain", "dense"): ([FNN_FWD], [FNN_BWD], [], "T-N"),
    ("fnn", "fused16", "bag", "dense"): ([BAG_FWD, BAG_FWD, FNN_FWD], [FNN_BWD, BAG_BWD, BAG_BWD], [], "T-N"),
    ("fnn", "split32", "plain", "dense"): ([FNN_FWD], [FNN_BWD], [], "TTN"),
    ("fnn", "split32", "bag", "dense"): ([BAG_FWD, BAG_FWD, FNN_FWD], [FNN_BWD, BAG_BWD, BAG_BWD], [], "TTN"),
    ("fnn", "fused16", "plain", "sgd"): ([FNN_FWD], [FNN_BWD], [], "N-N"),
    ("fnn", "fused16", "bag", "sgd"): ([BAG_FWD, BAG_FWD, FNN_FWD], [FNN_BWD, BAG_BWD, BAG_BWD], [], "N-N"),
    ("fnn", "split32", "plain", "sgd"): ([FNN_FWD], [FNN_BWD], [], "NNN"),
    ("fnn", "split32", "bag", "sgd"): ([BAG_FWD, BAG_FWD, FNN_FWD], [FNN_BWD, BAG_BWD, BAG_BWD], [], "NNN"),
    ("fnn", "fused16", "plain", "adam"): ([CATCH_UP, FNN_FWD], [], [ADVANCE, COUNT, ROWS_ADAM], "N-N"),
    ("fnn", "fused16", "bag", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FNN_FWD], [], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "N-N"),
    ("fnn", "split32", "plain", "adam"): ([CATCH_UP, FNN_FWD], [], [ADVANCE, COUNT, ROWS_ADAM], "NNN"),
    ("fnn", "split32", "bag", "adam"):
      ([CATCH_UP, CATCH_UP, BAG_FWD, BAG_FWD, FNN_FWD], [], [ADVANCE, COUNT, COUNT, ROWS_ADAM, ROWS_ADAM], "NNN"),
}


@pytest.mark.parametrize("kind,lookup,use,mode", EMBED_CASES)
def test_embedding_launch_plan(recorder, kind, lookup, use, mode):
    coll, opt = _collection(kind, mode)
    recorder.take()
    (fwd, bwd, step, grads), _ = _run_embed(coll, opt, recorder, use, _bags() if lookup == "bag" else None)
    assert (_names(fwd), _names(bwd), _names(step), grads) == PLANS["embed", kind, lookup, use, mode]


@pytest.mark.parametrize("lookup", ["plain", "bag"])
def test_no_grad_forward_catches_up_the_rows(recorder, lookup):
    coll, opt = _collection("fused16", "adam")
    recorder.take()
    with torch.no_grad():
        coll(_ids(), bags=_bags() if lookup == "bag" else None)
    assert _names(recorder.take()) == PLANS["no_grad", lookup]


@pytest.mark.parametrize("kind,lookup,mode", FNN_CASES)
def test_fnn_input_launch_plan(recorder, kind, lookup, mode):
    coll, opt = _collection(kind, mode)
    recorder.take()
    (fwd, bwd, step, grads), _ = _run_fnn(coll, opt, recorder, _bags() if lookup == "bag" else None)
    assert (_names(fwd), _names(bwd), _names(step), grads) == PLANS["fnn", kind, lookup, mode]


def _assert_close(got, want, what):
    assert (got is None) == (want is None), what
    if got is not None:
        # duplicate ids are summed with float atomics in a different order: absolute slack scaled to the tensor
        torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6 * float(want.abs().max()), msg=what)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", list(COLLECTIONS))
def test_bags_of_one_equal_the_plain_lookup(recorder, kind, mode):
    use = "stack" if kind == "nolin16" else "both"
    outs = []
    for bags in (None, _bags_of_one(_ids())):
        coll, opt = _collection(kind, mode)
        outs.append(_run_embed(coll, opt, recorder, use, bags)[1])
    plain, bag = outs
    assert plain.keys() == bag.keys()
    for key in plain:
        _assert_close(bag[key], plain[key], f"{kind} {mode}: {key}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["fused16", "split32"])
def test_fnn_bags_of_one_equal_the_plain_lookup(recorder, kind, mode):
    outs = []
    for bags in (None, _bags_of_one(_ids())):
        coll, opt = _collection(kind, mode)
        outs.append(_run_fnn(coll, opt, recorder, bags)[1])
    plain, bag = outs
    assert plain.keys() == bag.keys()
    for key in plain:
        _assert_close(bag[key], plain[key], f"{kind} {mode}: {key}")
