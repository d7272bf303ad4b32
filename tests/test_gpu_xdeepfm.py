"""GPU tests of the xDeepFM pieces outside the CIN kernels: the FM-free logit of the fused embedding kernel
(EmbeddingCollection.forward(second_order=False), DR_EMBED_NO_FM) and the XDeepFM model, one step against the float64
oracle composition (tests/cin_oracle.py), save / load and training through the Keras engine."""
import os
import tempfile

import numpy as np
import pytest
import torch

from cin_oracle import xdeepfm_forward

pytestmark = pytest.mark.gpu


def _ids(rng, B, rows, id_dtype, hot=True):
    """[B, S] ids with OOV ids (-1 and rows) and, with `hot`, one id repeated in half of the batch."""
    ids = np.stack([rng.integers(0, r, size=B) for r in rows], axis=1)
    ids[rng.random(ids.shape) < 0.05] = -1
    for s, r in enumerate(rows):
        ids[rng.random(B) < 0.03, s] = r
        if hot:
            ids[rng.random(B) < 0.5, s] = 1
    return torch.from_numpy(ids.astype(np.int64)).to("cuda", id_dtype)


@pytest.mark.parametrize("dim", [16, 32], ids=["fused-row-D16", "split-D32"])
@pytest.mark.parametrize("id_dtype", [torch.int64, torch.int32], ids=["i64", "i32"])
def test_second_order_false(dim, id_dtype):
    from deep_recommenders_b200.embedding import EmbeddingCollection
    rng = np.random.default_rng(dim)
    rows, B = [40, 7, 300, 1], 1000
    coll = EmbeddingCollection(rows, dim, with_linear=True, seed=1, device="cuda")
    with torch.no_grad():
        coll.lin_view().normal_(0, 0.5)
        coll.bias.fill_(0.25)
    ids = _ids(rng, B, rows, id_dtype)
    stack_fm, logit_fm = coll(ids)
    stack, logit = coll(ids, second_order=False)
    assert torch.equal(stack, stack_fm)                                   # the stack is bit-exact to the default path
    idn = ids.long().cpu().numpy()
    lin = [coll.linear_of(s).detach().double().cpu().numpy() for s in range(len(rows))]
    ref = np.full(B, 0.25)
    for s, r in enumerate(rows):
        ok = (idn[:, s] >= 0) & (idn[:, s] < r)
        ref[ok] += lin[s][idn[ok, s]]
    np.testing.assert_allclose(logit.detach().double().cpu().numpy(), ref, rtol=0, atol=1e-6)
    # backward: tables get g_stack only; first-order weights and bias still get g_logit
    gs = torch.randn(stack.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    gl = torch.randn(logit.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    torch.autograd.backward([stack, logit], [gs, gl])
    g_emb, g_lin, g_bias = coll.grads()
    gsn, gln = gs.double().cpu().numpy(), gl.double().cpu().numpy()
    for s, r in enumerate(rows):
        o = int(coll._offsets[s])
        ref_e, ref_l = np.zeros((r, dim)), np.zeros(r)
        ok = (idn[:, s] >= 0) & (idn[:, s] < r)
        np.add.at(ref_e, idn[ok, s], gsn[ok, s])
        np.add.at(ref_l, idn[ok, s], gln[ok])
        scale = np.zeros((r, dim))
        np.add.at(scale, idn[ok, s], np.abs(gsn[ok, s]))
        got_e = g_emb[o:o + r].double().cpu().numpy()
        assert np.all(np.abs(got_e - ref_e) <= 1e-6 * scale + 1e-12), s
        np.testing.assert_allclose(g_lin[o:o + r].double().cpu().numpy(), ref_l, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(float(g_bias), gln.sum(), rtol=1e-5, atol=1e-4)


def _model(rows, dim, **kw):
    from deep_recommenders.keras.layers import XDeepFM
    return XDeepFM(rows, dim, seed=3, device="cuda", **kw)


def _params64(m):
    """float64 CPU leaf copies of every model parameter (the embedding arena split into tables / first-order)."""
    c = m.embeddings
    P = {"emb": c.emb_view().detach().double().cpu().clone().requires_grad_(),
         "lin": c.lin_view().detach().double().cpu().clone().requires_grad_(),
         "bias": c.bias.detach().double().cpu().clone().requires_grad_()}
    for i, l in enumerate(m.cin):
        P[f"cin{i}"] = l.kernel.detach().double().cpu().clone().requires_grad_()
    for i, l in enumerate(m.dnn.layers):
        P[f"dw{i}"] = l.kernel.detach().double().cpu().clone().requires_grad_()
        P[f"db{i}"] = l.bias.detach().double().cpu().clone().requires_grad_()
    P["hw"] = m.head.kernel.detach().double().cpu().clone().requires_grad_()
    P["hb"] = m.head.bias.detach().double().cpu().clone().requires_grad_()
    return P


def _ref_logit(m, P, ids):
    """The same composition in float64 torch-CPU autograd (the gradients' oracle)."""
    c = m.embeddings
    ids = ids.long().cpu()
    B, S = ids.shape
    rows = torch.tensor(c.rows_list)
    ok = (ids >= 0) & (ids < rows)
    flat = torch.where(ok, ids + c._offsets.cpu(), torch.zeros_like(ids))
    x0 = P["emb"][flat] * ok[..., None]
    lin = P["bias"] + (P["lin"][flat] * ok).sum(1)
    x, pools = x0, []
    for i, l in enumerate(m.cin):
        w = P[f"cin{i}"].view(x0.shape[1], x.shape[1], -1)
        x = torch.sigmoid(torch.einsum("bid,bjd,ijk->bkd", x0, x, w))
        pools.append(x.sum(2))
    h = x0.reshape(B, -1)
    for i in range(len(m.dnn.layers)):
        h = torch.relu(h @ P[f"dw{i}"] + P[f"db{i}"])
    return (torch.cat(pools + [h], 1) @ P["hw"]).view(-1) + P["hb"] + lin


@pytest.mark.parametrize("id_dtype", [torch.int64, torch.int32], ids=["i64", "i32"])
def test_xdeepfm_step_matches_oracle(id_dtype):
    rng = np.random.default_rng(7)
    rows, dim, B = [60, 9, 400, 3, 25, 1000], 16, 700
    m = _model(rows, dim, cin_layers=(12, 7), dnn_units=(32, 8))
    with torch.no_grad():
        m.embeddings.lin_view().normal_(0, 0.3)
        m.embeddings.bias.fill_(-0.1)
    ids = _ids(rng, B, rows, id_dtype)
    y = torch.from_numpy((rng.random(B) < 0.3).astype(np.float32)).cuda()
    prob = m(ids).view(-1)
    loss = torch.nn.functional.binary_cross_entropy(prob, y)
    loss.backward()
    # forward against the numpy oracle
    c = m.embeddings
    tables = [c.table(s).detach().cpu().numpy() for s in range(len(rows))]
    lins = [c.linear_of(s).detach().cpu().numpy() for s in range(len(rows))]
    ref_prob, _ = xdeepfm_forward(tables, lins, float(c.bias.detach()), ids.long().cpu().numpy(),
                                  [l.kernel.detach().cpu().numpy() for l in m.cin], "sigmoid",
                                  [l.kernel.detach().cpu().numpy() for l in m.dnn.layers],
                                  [l.bias.detach().cpu().numpy() for l in m.dnn.layers], "relu",
                                  m.head.kernel.detach().cpu().numpy(), m.head.bias.detach().cpu().numpy())
    np.testing.assert_allclose(prob.detach().double().cpu().numpy(), ref_prob, rtol=1e-5, atol=1e-6)
    # loss and every gradient against float64 autograd of the same composition
    P = _params64(m)
    z = _ref_logit(m, P, ids)
    ref_loss = torch.nn.functional.binary_cross_entropy_with_logits(z, y.double().cpu())
    ref_loss.backward()
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    g_emb, g_lin, g_bias = c.grads()
    got = {"emb": g_emb, "lin": g_lin, "bias": g_bias, "hw": m.head.kernel.grad, "hb": m.head.bias.grad}
    for i, l in enumerate(m.cin):
        got[f"cin{i}"] = l.kernel.grad
    for i, l in enumerate(m.dnn.layers):
        got[f"dw{i}"], got[f"db{i}"] = l.kernel.grad, l.bias.grad
    for k, g in got.items():
        ref = P[k].grad.numpy()
        tol = 1e-4 * max(np.abs(ref).max(), 1e-6)
        np.testing.assert_allclose(g.detach().double().cpu().numpy().reshape(ref.shape), ref, rtol=1e-4, atol=tol,
                                   err_msg=k)


def test_xdeepfm_save_load_and_config():
    rows, dim = [50, 20, 80], 8
    m = _model(rows, dim, cin_layers=(6, 4), dnn_units=(16,))
    ids = _ids(np.random.default_rng(1), 64, rows, torch.int64)
    pred = m.predict(ids)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "xdeepfm.pt")
        m.save(path)
        blob = torch.load(path, weights_only=False)
        from deep_recommenders.keras.layers import XDeepFM
        cfg = {k: v for k, v in blob["config"].items() if k not in ("name", "trainable", "dtype")}
        loaded = XDeepFM(**cfg, device="cuda")
        loaded(ids)
        loaded.load_state_dict(blob["state"])
        assert loaded.get_config() == m.get_config()
        assert torch.equal(loaded.predict(ids), pred)


def test_xdeepfm_fit_through_keras_engine():
    rows, dim, B = [100, 30, 200, 50], 16, 512
    m = _model(rows, dim, cin_layers=(16, 16), dnn_units=(32, 8))
    rng = np.random.default_rng(2)
    ids = _ids(rng, B, rows, torch.int64, hot=False)
    y = torch.from_numpy((ids[:, 0].cpu().numpy() % 2).astype(np.float32)).cuda()
    m.compile(loss="binary_crossentropy", optimizer="adam")
    hist = m.fit(ids, y, epochs=8, steps_per_epoch=1)
    losses = hist["loss"]
    assert np.all(np.isfinite(losses)) and losses[-1] < losses[0], losses
