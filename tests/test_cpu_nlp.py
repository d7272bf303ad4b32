"""CPU checks of the Transformer port (no GPU): the numpy oracle against the golden vectors made by executing the
reference's own multi_head_attention.py and transformer.py, the padding constant's known answers, the oracle's
gradients against torch autograd, errors raised before any CUDA call, config round trips, the engine's new loss and
callback hooks, and host-side C-ABI validation."""
import os

import numpy as np
import pytest
import torch

import nlp_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "nlp_golden.npz")


@pytest.mark.parametrize("pre,dtype", [("f64_", np.float64), ("f32_", np.float32)])
def test_oracle_reproduces_golden(pre, dtype):
    """The reference's ScaledDotProductAttention casts its inputs to float32 (:68-70): its outputs are float32 results
    in both files, so the float64 oracle meets them within float32 rounding, fully padded rows (uniform) included."""
    g = np.load(GOLDEN)
    n = 0
    for key in [k[:-4] for k in g.files if k.startswith(pre + "sdpa_") and k.endswith("_out")]:
        mask = g[key + "_mask"] if bool(g[key + "_masking"]) else None
        got = O.attention(g[key + "_q"], g[key + "_k"], g[key + "_v"], mask, 1, bool(g[key + "_future"]))
        np.testing.assert_allclose(got, g[key + "_out"], rtol=1e-5, atol=1e-6, err_msg=key)
        n += 1
    for key in [k[:-4] for k in g.files if k.startswith(pre + "mha_") and k.endswith("_out")]:
        H = int(g[key + "_heads"])
        mask = g[key + "_mask"] if bool(g[key + "_masking"]) else None
        q, k, v = (g[key + n_] @ g[key + w] for n_, w in (("_q", "_wq"), ("_k", "_wk"), ("_v", "_wv")))
        got = O.attention(q, k, v, mask, H, bool(g[key + "_future"]))
        np.testing.assert_allclose(got, g[key + "_out"], rtol=1e-5, atol=1e-6, err_msg=key)
        n += 1
    assert n == 12
    tol = 1e-12 if dtype == np.float64 else 2e-6
    np.testing.assert_allclose(O.layer_norm(g[pre + "ln_x"], None, g[pre + "ln_gamma"], g[pre + "ln_beta"],
                                            dtype=dtype), g[pre + "ln_out"], rtol=tol * 10, atol=tol * 10)
    L, d = (int(s) for s in g[pre + "pe_shape"][1:3])
    np.testing.assert_array_equal(O.position_encoding(L, d).astype(np.float32), g[pre + "pe_out"])
    w = {k[len(pre + "tr_w_"):]: g[k] for k in g.files if k.startswith(pre + "tr_w_")}
    got = O.transformer(w, g[pre + "tr_enc"], g[pre + "tr_dec"], 2)
    np.testing.assert_allclose(got, g[pre + "tr_out"], rtol=1e-4, atol=1e-6)


def test_padding_constant_known_answers():
    rng = np.random.default_rng(0)
    q, k, v = (rng.standard_normal((2, 6, 4)) for _ in range(3))
    mask = np.zeros((2, 6), np.float32)
    mask[0] = 1.0
    out = O.attention(q, k, v, mask)
    np.testing.assert_allclose(out[0], np.broadcast_to(v[0].mean(0), (6, 4)), rtol=1e-12)
    mask = np.zeros((2, 6), np.float32)
    mask[:, 0] = 1.0
    out = O.attention(q, k, v, mask, causal=True)
    np.testing.assert_allclose(out[:, 0], v.mean(1), rtol=1e-12)          # row 0 spans the future keys too
    # the other rows of the causal case see keys 1..i only
    p = O.softmax(O.scores(q, k, mask, True)[0])
    assert np.all(p[:, 1:][np.triu(np.ones((5, 6), bool), 2)[None].repeat(2, 0)] == 0)


def _torch_attention(q, k, v, mask, H, causal, rate, seed):
    qs, ks, vs = (torch.from_numpy(O.split_heads(x, H)) for x in (q, k, v))
    div = float(np.float32(np.sqrt(qs.shape[-1])))
    s = qs @ ks.transpose(1, 2) / div
    if mask is not None:
        m = torch.from_numpy(np.tile(mask, (qs.shape[0] // mask.shape[0], 1))[:, None, :]).double()
        s = s + m * float(O.NEG)
    if causal:
        s = torch.where(torch.triu(torch.ones(s.shape[1:], dtype=torch.bool), 1), torch.full_like(s, float(O.NEG)), s)
    p = torch.softmax(s, -1)
    if rate > 0:
        p = p * float(O.keep_scale(rate)) * torch.from_numpy(O.keep_mask(seed, rate, *s.shape)).double()
    return p @ vs


@pytest.mark.parametrize("mask_kind,causal,rate", [("none", False, 0.0), ("pad", False, 0.0), ("pad", True, 0.0),
                                                   ("none", True, 0.3), ("pad", False, 0.5)])
def test_attention_grad_matches_torch_autograd(mask_kind, causal, rate):
    rng = np.random.default_rng(1)
    B, H, L, dh = 3, 2, 7, 3
    q, k, v, g = (rng.standard_normal((B, L, H * dh)) for _ in range(4))
    mask = (rng.random((B, L)) < 0.3).astype(np.float32) if mask_kind == "pad" else None
    tq, tk, tv = (torch.from_numpy(x).requires_grad_() for x in (q, k, v))
    out = _torch_attention(tq.detach().numpy(), tk.detach().numpy(), tv.detach().numpy(), mask, H, causal, rate, 9)
    np.testing.assert_allclose(O.merge_heads(out.numpy(), H), O.attention(q, k, v, mask, H, causal, rate, 9),
                               rtol=1e-10, atol=1e-12)
    # torch autograd through the head split
    qs, ks, vs = (x.reshape(B, L, H, dh).permute(2, 0, 1, 3).reshape(H * B, L, dh) for x in (tq, tk, tv))
    div = float(np.float32(np.sqrt(dh)))
    s = qs @ ks.transpose(1, 2) / div
    if mask is not None:
        s = s + torch.from_numpy(np.tile(mask, (H, 1))[:, None, :]).double() * float(O.NEG)
    if causal:
        s = torch.where(torch.triu(torch.ones(L, L, dtype=torch.bool), 1), torch.full_like(s, float(O.NEG)), s)
    p = torch.softmax(s, -1)
    if rate > 0:
        p = p * float(O.keep_scale(rate)) * torch.from_numpy(O.keep_mask(9, rate, H * B, L, L)).double()
    o = (p @ vs).reshape(H, B, L, dh).permute(1, 2, 0, 3).reshape(B, L, H * dh)
    o.backward(torch.from_numpy(g))
    for got, t in zip(O.attention_grad(q, k, v, g, mask, H, causal, rate, 9), (tq, tk, tv)):
        np.testing.assert_allclose(got, t.grad.numpy(), rtol=1e-9, atol=1e-11)


def test_mask_gradient_rules():
    """A fully padded row passes gradient to q and k (the add keeps it); a causal-replaced score passes none."""
    rng = np.random.default_rng(2)
    q, k, v, g = (rng.standard_normal((1, 5, 3)) for _ in range(4))
    mask = np.ones((1, 5), np.float32)
    gq, gk, _ = O.attention_grad(q, k, v, g, mask)
    assert np.abs(gq).max() > 0 and np.abs(gk).max() > 0
    # causal: query 0 with every key padded has uniform p over all keys, but the replaced keys 1..4 give gk nothing
    mask = np.zeros((1, 5), np.float32)
    mask[0, 0] = 1.0
    q1 = np.zeros_like(q)
    q1[0, 0] = q[0, 0]
    g1 = np.zeros_like(g)
    g1[0, 0] = g[0, 0]
    gq, gk, gv = O.attention_grad(q1, k, v, g1, mask, causal=True)
    assert np.all(gk[0, 1:] == 0) and np.all(np.abs(gv[0]) > 0)


def test_layer_norm_and_softmax_grads_match_torch_autograd():
    rng = np.random.default_rng(3)
    x, r, gy = (rng.standard_normal((4, 6)) for _ in range(3))
    gamma, beta = rng.standard_normal(6), rng.standard_normal(6)
    tx, tr, tg, tb = (torch.from_numpy(a).requires_grad_() for a in (x, r, gamma, beta))
    s = tx + tr
    mu = s.mean(-1, keepdim=True)
    var = ((s - mu.detach()) ** 2).mean(-1, keepdim=True)        # tf.nn.moments stops the mean's gradient
    y = tg * ((s - mu) / (var + 1e-8) ** 0.5) + tb
    np.testing.assert_allclose(y.detach().numpy(), O.layer_norm(x, r, gamma, beta), rtol=1e-12)
    y.backward(torch.from_numpy(gy))
    gx, gg, gb = O.layer_norm_grad(x, r, gamma, gy)
    np.testing.assert_allclose(gx, tx.grad.numpy(), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(gx, tr.grad.numpy(), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(gg, tg.grad.numpy(), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(gb, tb.grad.numpy(), rtol=1e-9, atol=1e-11)
    tx = torch.from_numpy(x).requires_grad_()
    ys = torch.softmax(tx, -1)
    ys.backward(torch.from_numpy(gy))
    np.testing.assert_allclose(O.softmax_grad(ys.detach().numpy(), gy), tx.grad.numpy(), rtol=1e-9, atol=1e-12)


def test_keep_mask_is_stateless_and_rate_dependent():
    a = O.keep_mask(5, 0.25, 2, 3, 4)
    assert np.array_equal(a, O.keep_mask(5, 0.25, 2, 3, 4))
    assert not np.array_equal(a, O.keep_mask(6, 0.25, 2, 3, 4))
    assert O.keep_mask(5, 0.0, 2, 3, 4).all()
    big = O.keep_mask(123, 0.4, 4, 64, 64)
    n = big.size
    assert abs(big.sum() - 0.6 * n) < 5 * np.sqrt(n * 0.24)


def test_layer_errors_before_any_cuda_call(monkeypatch):
    from deep_recommenders_b200 import _lib
    from deep_recommenders.keras.models.nlp import multi_head_attention as M
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    monkeypatch.setattr(_lib, "load", lambda: pytest.fail("C-ABI reached"))
    x = torch.zeros((2, 3, 4))
    with pytest.raises(AssertionError, match=r"inputs should be set \[queries, keys, values, masks\]."):
        M.ScaledDotProductAttention()([x, x, x])
    with pytest.raises(AssertionError, match=r"inputs should be set \[queries, keys, values\]."):
        M.ScaledDotProductAttention(masking=False)([x, x, x, x])
    with pytest.raises(AssertionError, match="masks"):
        M.MultiHeadAttention(2, 2)([x, x, x])
    with pytest.raises(ValueError, match="same length"):
        M.ScaledDotProductAttention(masking=False, future=True)([x, torch.zeros((2, 5, 4)), torch.zeros((2, 5, 4))])
    with pytest.raises(ValueError, match="same length"):
        M.MultiHeadAttention(2, 2, masking=False, future=True, seed=0)([x, torch.zeros((2, 5, 4)),
                                                                        torch.zeros((2, 5, 4))])


def test_config_round_trips():
    from deep_recommenders.keras.models.nlp import MultiHeadAttention, Transformer
    from deep_recommenders.keras.models.nlp import multi_head_attention as M, transformer as T
    g = np.load(GOLDEN)
    tr_keys = {str(k) for k in g["f64_tr_config_keys"]}
    t = Transformer(50, 8, n_heads=2, encoder_stack=1, decoder_stack=3, feed_forward_size=16, dropout_rate=0.2)
    cfg = t.get_config()
    assert tr_keys <= set(cfg)
    assert Transformer.from_config(cfg).get_config() == cfg
    m = MultiHeadAttention(4, 8, dropout_rate=0.3, masking=False, future=True, trainable=False)
    cfg = m.get_config()
    assert {"n_heads", "head_dim", "dropout_rate", "masking", "future", "trainable"} <= set(cfg)
    assert MultiHeadAttention.from_config(cfg).get_config() == cfg
    for layer in (M.ScaledDotProductAttention(masking=False, future=True, dropout_rate=0.1), M.Embedding(10, 4),
                  T.PositionEncoding(8), T.PositionWiseFeedForward(8, 16), T.LayerNormalization(1e-6), T.Add()):
        cfg = layer.get_config()
        assert type(layer).from_config(cfg).get_config() == cfg


def test_reference_import_paths():
    from deep_recommenders.keras.models.nlp import MultiHeadAttention, Transformer
    from deep_recommenders.keras.models.nlp.multi_head_attention import MultiHeadAttention as M2
    from deep_recommenders.keras.models.nlp.transformer import Noam, Transformer as T2, label_smoothing
    assert MultiHeadAttention is M2 and Transformer is T2 and Noam is not None
    np.testing.assert_allclose(label_smoothing(np.eye(4)), 0.9 * np.eye(4) + 0.025)


def test_categorical_crossentropy_registered():
    from deep_recommenders_b200.keras import engine
    yt = torch.tensor([[0.0, 1.0], [1.0, 0.0]])
    yp = torch.tensor([[0.2, 0.8], [0.5, 0.5]])
    np.testing.assert_allclose(engine._LOSSES["categorical_crossentropy"](yt, yp).numpy(),
                               [-np.log(0.8), -np.log(0.5)], rtol=1e-6)


def test_noam_drives_the_learning_rate_through_the_engine():
    from deep_recommenders_b200.keras import engine
    from deep_recommenders.keras.layers import Model
    from deep_recommenders.keras.models.nlp.transformer import Noam

    class Tiny(Model):          # a CPU torch model: only the engine's hooks are under test
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(3))
            self.built = True

        def call(self, x, **kwargs):
            return torch.sigmoid(x @ self.w).reshape(-1, 1)

    m = Tiny().compile(loss="binary_crossentropy", optimizer=engine.Adam())
    seen = []

    class Spy:
        def on_epoch_end(self, epoch, logs):
            seen.append(m.optimizer.lr)
            return False

    noam = Noam(model_dim=16, warmup_steps=10)
    data = [(torch.ones((4, 3)), torch.ones(4))] * 6
    m.fit(iter(data), epochs=2, steps_per_epoch=3, callbacks=[Spy(), noam, engine.EarlyStopping(patience=5)])
    assert noam._step_num == 6
    assert seen == pytest.approx([16 ** -.5 * 3 * 10 ** -1.5, 16 ** -.5 * 6 * 10 ** -1.5])
    assert m._optimizer.param_groups[0]["lr"] == pytest.approx(16 ** -.5 * 6 * 10 ** -1.5)


def test_c_abi_host_validation(lib):
    p = 256
    #                   q  k  v  mask B  H  Lq Lk dh Bm causal rate seed out lse stream
    assert lib.dr_mha_attn_fwd(None, p, p, None, 2, 1, 4, 4, 8, 0, 0, 0.0, 0, p, p, None) == -1
    assert b"null pointer" in lib.dr_last_error()
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 4, 4, 8, 0, 0, 0.0, 0, p, None, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, -1, 1, 4, 4, 8, 0, 0, 0.0, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 0, 4, 4, 8, 0, 0, 0.0, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 0, 4, 8, 0, 0, 0.0, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 4, 4, 0, 0, 0, 0.0, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, p, 2, 3, 4, 4, 8, 4, 0, 0.0, 0, p, p, None) == -1   # Bm does not divide
    assert b"divide" in lib.dr_last_error()
    assert lib.dr_mha_attn_fwd(p, p, p, p, 2, 3, 4, 4, 8, 0, 0, 0.0, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 4, 5, 8, 0, 1, 0.0, 0, p, p, None) == -1  # causal, Lq != Lk
    assert b"causal" in lib.dr_last_error()
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 4, 4, 8, 0, 0, 1.0, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 4, 4, 8, 0, 0, -0.1, 0, p, p, None) == -1
    assert lib.dr_mha_attn_fwd(p, p, p, None, 2, 1, 4, 4, 129, 0, 0, 0.0, 0, p, p, None) == -3
    assert lib.dr_mha_attn_fwd(p, p, p, None, 1 << 20, 8, 1 << 8, 4, 8, 0, 0, 0.0, 0, p, p, None) == -3
    assert lib.dr_mha_attn_fwd(None, None, None, None, 0, 1, 4, 4, 8, 0, 0, 0.0, 0, None, None, None) == 0
    # backward: q k v mask out lse g_out B H Lq Lk dh Bm causal rate seed gq gk gv stream
    assert lib.dr_mha_attn_bwd(p, p, p, None, p, p, None, 2, 1, 4, 4, 8, 0, 0, 0.0, 0, p, p, p, None) == -1
    assert lib.dr_mha_attn_bwd(p, p, p, None, p, p, p, 2, 1, 4, 4, 8, 0, 0, 0.0, 0, p, None, p, None) == -1
    assert lib.dr_mha_attn_bwd(p, p, p, None, p, p, p, 2, 1, 4, 4, 200, 0, 0, 0.0, 0, p, p, p, None) == -3
    assert lib.dr_mha_attn_bwd(p, p, p, None, p, p, p, 2, 1, 3, 4, 8, 0, 1, 0.0, 0, p, p, p, None) == -1
    # LayerNorm, softmax
    assert lib.dr_add_layernorm_fwd(p, None, None, p, 4, 8, 1e-8, p, None) == -1
    assert lib.dr_add_layernorm_fwd(p, None, p, p, 4, 0, 1e-8, p, None) == -1
    assert lib.dr_add_layernorm_fwd(None, None, p, p, 0, 8, 1e-8, None, None) == 0
    assert lib.dr_add_layernorm_bwd(p, None, p, p, 4, 8, 1e-8, p, None, p, None) == -1
    assert lib.dr_add_layernorm_bwd(p, None, p, p, 4, 5000, 1e-8, p, p, p, None) == -3
    assert lib.dr_softmax_rows_fwd(None, 4, 8, p, None) == -1
    assert lib.dr_softmax_rows_fwd(p, 4, 0, p, None) == -1
    assert lib.dr_softmax_rows_bwd(p, None, 4, 8, p, None) == -1
    assert lib.dr_softmax_rows_fwd(None, 0, 8, None, None) == 0
