"""Rows R, R1, R2, R3 on the GPU through the C-ABI against the numpy oracle, plus the reference's
seeded property tests ported: tests/keras/test_sbcnm.py:16-41 and :43-55."""
import numpy as np
import pytest
import torch

from oracle import reference_np as R

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


CASES = [
    # nq, nc, D, tau, weights, probs, ids
    (1, 1, 4, None, False, False, False),
    (8, 8, 16, None, False, False, False),
    (70, 70, 64, 0.5, True, False, False),
    (64, 130, 32, None, False, True, False),
    (130, 130, 64, 0.2, True, True, True),
    (257, 300, 128, None, True, True, True),
    (100, 100, 8, 2.0, False, False, True),
    (65, 65, 200, None, False, False, False),
]


@pytest.mark.parametrize("nq,nc,D,tau,use_w,use_p,use_ids", CASES)
def test_inbatch_softmax_loss_and_grads(nq, nc, D, tau, use_w, use_p, use_ids):
    from deep_recommenders.keras.models.retrieval import sbcnm
    rng = np.random.default_rng(nq + nc + D)
    q = (rng.standard_normal((nq, D)) / np.sqrt(D) * 3).astype(np.float32)
    c = (rng.standard_normal((nc, D)) / np.sqrt(D) * 3).astype(np.float32)
    w = rng.uniform(0.5, 2.0, nq).astype(np.float32) if use_w else None
    p = rng.uniform(0.01, 1.0, nc).astype(np.float32) if use_p else None
    ids = rng.integers(0, max(2, nc // 3), nc).astype(np.int64) if use_ids else None
    qt, ct = cu(q).requires_grad_(True), cu(c).requires_grad_(True)
    task = sbcnm.Retrieval(temperature=tau)
    loss = task(qt, ct, sample_weight=None if w is None else cu(w),
                candidate_sampling_probability=None if p is None else cu(p),
                candidate_ids=None if ids is None else cu(ids))
    (loss * 1.5).backward()
    ref_loss, _, _ = R.retrieval_loss(q, c, w, p, ids, tau, None, np.float64)
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)) + 1e-4
    gq, gc = R.retrieval_grad(q, c, w, p, ids, tau, np.float64)
    gq, gc = 1.5 * gq, 1.5 * gc
    assert np.abs(qt.grad.cpu().numpy() - gq).max() <= 2e-5 * np.abs(gq).max() + 1e-6
    assert np.abs(ct.grad.cpu().numpy() - gc).max() <= 2e-5 * np.abs(gc).max() + 1e-6


def test_scores_kernel_matches_helper_layers():
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(0)
    q = rng.standard_normal((37, 24)).astype(np.float32)
    c = rng.standard_normal((53, 24)).astype(np.float32)
    p = rng.uniform(0.05, 1, 53).astype(np.float32)
    ids = rng.integers(0, 10, 53).astype(np.int64)
    s = ops.scores(cu(q), cu(c), cu(p), cu(ids)).cpu().numpy()
    ref = q.astype(np.float64) @ c.astype(np.float64).T
    ref = R.sampling_probability_correction(ref, p.astype(np.float64))
    ref = R.remove_accidental_negative(ref, np.eye(37, 53), ids)
    big = np.abs(ref) > 1e30
    assert np.array_equal(big, np.abs(s) > 1e30)
    assert np.allclose(s[~big], ref[~big], rtol=1e-5, atol=1e-5)
    assert np.allclose(s[big], R.MIN_FLOAT, rtol=1e-5)


@pytest.mark.parametrize("num_hard_negatives", [3, 5, 10, 15])
def test_ref_hard_negative_mining(num_hard_negatives):
    """tests/keras/test_sbcnm.py:16-41."""
    from deep_recommenders.keras.models.retrieval import sbcnm
    logits_shape = (2, 20)
    rng = np.random.RandomState(42)
    logits = rng.uniform(size=logits_shape).astype(np.float32)
    labels = rng.permutation(np.eye(*logits_shape).T).T.astype(np.float32)
    out_logits, out_labels = sbcnm.HardNegativeMining(num_hard_negatives)(cu(logits), cu(labels))
    assert out_logits.shape[-1] == num_hard_negatives + 1
    assert np.allclose((out_logits * out_labels).sum(-1).cpu().numpy(), (logits * labels).sum(-1))
    logits = logits + labels * 1000.0
    out_logits, out_labels = sbcnm.HardNegativeMining(num_hard_negatives)(cu(logits), cu(labels))
    out_logits, out_labels = out_logits.cpu().numpy(), out_labels.cpu().numpy()
    assert np.allclose(np.sort(logits, axis=1)[:, -num_hard_negatives - 1:], np.sort(out_logits))


def test_ref_remove_accidental_negative():
    """tests/keras/test_sbcnm.py:43-55."""
    from deep_recommenders.keras.models.retrieval import sbcnm
    logits_shape = (2, 4)
    rng = np.random.RandomState(42)
    logits = rng.uniform(size=logits_shape).astype(np.float32)
    labels = rng.permutation(np.eye(*logits_shape).T).T.astype(np.float32)
    identifiers = rng.randint(0, 3, size=logits_shape[-1])
    out_logits = sbcnm.RemoveAccidentalNegative()(cu(logits), cu(labels), cu(identifiers))
    assert np.allclose((out_logits * cu(labels)).sum(1).cpu().numpy(), (logits * labels).sum(1))
    assert np.allclose(out_logits.cpu().numpy(), R.remove_accidental_negative(logits, labels, identifiers))


@pytest.mark.parametrize("nq,k", [(20, 3), (64, 10), (100, 99)])
def test_hard_negative_topk_kernel_inbatch(nq, k):
    from deep_recommenders.keras.models.retrieval import sbcnm
    rng = np.random.default_rng(nq)
    logits = rng.standard_normal((nq, nq)).astype(np.float32)
    labels = np.eye(nq, dtype=np.float32)
    ol, oy = sbcnm.HardNegativeMining(k)(cu(logits), cu(labels))
    rl, ry, _ = R.hard_negative_mining(logits, labels, k)
    assert np.array_equal(np.sort(ol.cpu().numpy(), axis=1), np.sort(rl, axis=1))
    assert np.array_equal(oy.cpu().numpy().sum(1), np.ones(nq))


def test_retrieval_with_hard_negatives_matches_oracle():
    from deep_recommenders.keras.models.retrieval import sbcnm
    rng = np.random.default_rng(5)
    q = rng.standard_normal((48, 32)).astype(np.float32)
    c = rng.standard_normal((48, 32)).astype(np.float32)
    qt, ct = cu(q).requires_grad_(True), cu(c).requires_grad_(True)
    loss = sbcnm.Retrieval(temperature=0.7, num_hard_negatives=5)(qt, ct)
    ref, _, _ = R.retrieval_loss(q, c, None, None, None, 0.7, 5, np.float64)
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)) + 1e-4
    loss.backward()
    assert torch.isfinite(qt.grad).all() and torch.isfinite(ct.grad).all()


def test_full_size_c4_properties():
    """BASELINE config C4 (B=16384, D=64): loss equals the blockwise torch float64 evaluation; the
    gradient rows of softmax - eye sum to zero (sum_j G_ij = 0) => gQ . 1-projection identity."""
    from deep_recommenders.keras.models.retrieval import sbcnm
    B, D = 16384, 64
    gen = torch.Generator(device="cuda").manual_seed(0)
    q = (torch.randn(B, D, device="cuda", generator=gen) * 0.3).requires_grad_(True)
    c = (torch.randn(B, D, device="cuda", generator=gen) * 0.3).requires_grad_(True)
    loss = sbcnm.Retrieval()(q, c)
    loss.backward()
    ref = torch.zeros((), dtype=torch.float64, device="cuda")
    cs = c.detach().double()
    for i in range(0, B, 2048):
        s = q.detach()[i:i + 2048].double() @ cs.T
        ref += (torch.logsumexp(s, 1) - s[torch.arange(s.shape[0]), torch.arange(i, i + s.shape[0])]).sum()
    assert abs(float(loss) - float(ref)) <= 1e-5 * float(ref)
    # sum_i gC_i = sum_i sum_j G_ji q_j ... use: sum over all of gQ == sum_j (colsum G)_j c_j; and rows of G sum to 0
    # => gQ_i = sum_j P_ij c_j - c_i, so  sum_i gQ_i + sum_i c_i = sum_j (sum_i P_ij) c_j ; check against gC identity:
    # sum_j gC_j = sum_i (sum_j G_ij) q_i = 0
    # (cancellation-aware bound: 1e-5 of the sum of |terms| of each column sum)
    assert float((c.grad.double().sum(0).abs() / c.grad.double().abs().sum(0)).max()) <= 1e-5


@pytest.mark.parametrize("nq,nc,D,tau,use_w,use_p,use_ids,ws_bytes", [
    (130, 130, 64, 0.2, True, True, True, 2 << 30),       # one score block
    (257, 300, 128, None, True, True, True, 2 << 30),
    (513, 513, 64, 0.5, True, False, True, 128 * 513 * 4),    # query rows in blocks of 128 (backward recomputes scores)
    (300, 300, 32, None, False, False, False, 128 * 300 * 4),
    (64, 130, 32, None, False, True, False, 2 << 30),
])
def test_inbatch_softmax_tensor_core_form(nq, nc, D, tau, use_w, use_p, use_ids, ws_bytes):
    """The tensor-core form (dr_inbatch_softmax_fwd_ws / _bwd_ws: score blocks through the 3xTF32 GEMM core) against the
    float64 oracle and against the fused FFMA kernels -- forced on at sizes the default heuristic gives to the latter."""
    from deep_recommenders.keras.models.retrieval import sbcnm
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(nq + nc + D + 1)
    q = (rng.standard_normal((nq, D)) / np.sqrt(D) * 3).astype(np.float32)
    c = (rng.standard_normal((nc, D)) / np.sqrt(D) * 3).astype(np.float32)
    w = rng.uniform(0.5, 2.0, nq).astype(np.float32) if use_w else None
    p = rng.uniform(0.01, 1.0, nc).astype(np.float32) if use_p else None
    ids = rng.integers(0, max(2, nc // 3), nc).astype(np.int64) if use_ids else None
    task = sbcnm.Retrieval(temperature=tau)
    kw = dict(sample_weight=None if w is None else cu(w), candidate_sampling_probability=None if p is None else cu(p),
              candidate_ids=None if ids is None else cu(ids))
    out = {}
    old = (ops.SOFTMAX_TC_MIN_SCORES, ops.SOFTMAX_TC_WS_BYTES)
    try:
        for form, min_scores in (("tc", 0), ("ffma", 1 << 62)):
            ops.SOFTMAX_TC_MIN_SCORES, ops.SOFTMAX_TC_WS_BYTES = min_scores, ws_bytes
            qt, ct = cu(q).requires_grad_(True), cu(c).requires_grad_(True)
            loss = task(qt, ct, **kw)
            (loss * 1.5).backward()
            out[form] = (float(loss), qt.grad.cpu().numpy(), ct.grad.cpu().numpy())
    finally:
        ops.SOFTMAX_TC_MIN_SCORES, ops.SOFTMAX_TC_WS_BYTES = old
    ref_loss, _, _ = R.retrieval_loss(q, c, w, p, ids, tau, None, np.float64)
    gq, gc = R.retrieval_grad(q, c, w, p, ids, tau, np.float64)
    gq, gc = 1.5 * gq, 1.5 * gc
    for form in ("tc", "ffma"):
        l, a, b = out[form]
        assert abs(l - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)) + 1e-4, form
        assert np.abs(a - gq).max() <= 2e-5 * np.abs(gq).max() + 1e-6, form
        assert np.abs(b - gc).max() <= 2e-5 * np.abs(gc).max() + 1e-6, form
