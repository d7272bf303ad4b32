"""GPU tests of the Transformer kernels (dr_mha_attn_fwd / _bwd, dr_add_layernorm_fwd / _bwd, dr_softmax_rows_fwd /
_bwd), the nlp layers and a whole Transformer.

Every fp32 result must sit within 1e-5 x (sum of |terms|) of a float64 reference, where a score's own rounding is
carried into the terms that use it; outputs are written between sentinel guards so a store outside them is caught."""
import os
import tempfile
import zlib

import numpy as np
import pytest
import torch

import nlp_oracle as O

pytestmark = pytest.mark.gpu
SENT = 1234.5
PAD = 4099


def _lib():
    from deep_recommenders_b200 import _lib
    return _lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n, dtype=torch.float32):
    full = torch.full((n + 2 * PAD,), SENT, device="cuda", dtype=dtype)
    return full, full[PAD:PAD + n]


def _check_guards(full, n):
    f = full.cpu().numpy()
    assert np.all(f[:PAD] == SENT) and np.all(f[PAD + n:] == SENT), "store outside the output"


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _close(got, ref, scale, what, rel=1e-5):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    bound = rel * scale + 4.8e-7 * np.abs(ref) + 1e-30
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} out of bound; worst err {err.max():.3g}, "
                           f"bound there {bound.reshape(-1)[np.argmax((err - bound).reshape(-1))]:.3g}")


def attn_fwd(q, k, v, mask, H, causal, rate=0.0, seed=0):
    B, Lq, HD = q.shape
    Lk = k.shape[1]
    ofull, o = _guarded(q.numel())
    lfull, lse = _guarded(H * B * Lq, torch.float64)
    Bm = 0 if mask is None else mask.shape[0]
    rc = _lib().dr_mha_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), None if mask is None else mask.data_ptr(),
                                B, H, Lq, Lk, HD // H, Bm, int(causal), rate, seed, o.data_ptr(), lse.data_ptr(),
                                _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    _check_guards(ofull, q.numel())
    _check_guards(lfull, H * B * Lq)
    return o.view(B, Lq, HD), lse


def attn_bwd(q, k, v, mask, out, lse, g, H, causal, rate=0.0, seed=0):
    B, Lq, HD = q.shape
    Lk = k.shape[1]
    bufs = [_guarded(q.numel()), _guarded(k.numel()), _guarded(v.numel())]
    Bm = 0 if mask is None else mask.shape[0]
    rc = _lib().dr_mha_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), None if mask is None else mask.data_ptr(),
                                out.data_ptr(), lse.data_ptr(), g.data_ptr(), B, H, Lq, Lk, HD // H, Bm, int(causal),
                                rate, seed, *(b[1].data_ptr() for b in bufs), _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    for (full, t) in bufs:
        _check_guards(full, t.numel())
    return bufs[0][1].view(q.shape), bufs[1][1].view(k.shape), bufs[2][1].view(v.shape)


def _abs_terms(q, k, v, g, mask, H, causal, rate, seed):
    """Sums of |terms| of out, gq, gk, gv (float64), with each score's rounding (1 + sum |q||k| / div) carried on."""
    qs, ks, vs, gs = (np.abs(O.split_heads(np.asarray(x, np.float64), H)) for x in (q, k, v, g))
    s, _ = O.scores(O.split_heads(q, H), O.split_heads(k, H), mask, causal)
    p = O.softmax(s)
    div = np.float64(np.float32(np.sqrt(qs.shape[-1])))
    sa = 1.0 + np.einsum("rid,rjd->rij", qs, ks) / div
    kp = O.keep_mask(seed, rate, *s.shape) * np.float64(O.keep_scale(rate)) if rate > 0 else 1.0
    pa = p * sa * (kp if rate > 0 else 1.0) + p * sa
    out = np.einsum("rij,rjd->rid", pa, vs)
    dpa = np.einsum("rid,rjd->rij", gs, vs) * (kp if rate > 0 else 1.0)
    Da = (p * sa * dpa).sum(-1, keepdims=True)
    dsa = p * sa * (dpa + Da)
    gq = np.einsum("rij,rjd->rid", dsa, ks) / div
    gk = np.einsum("rij,rid->rjd", dsa, qs) / div
    gv = np.einsum("rij,rid->rjd", pa, gs)
    return tuple(O.merge_heads(x, H) for x in (out, gq, gk, gv))


def _mask(rng, kind, B, H, Lk, Bm):
    if kind == "none":
        return None
    m = (rng.random((Bm, Lk)) < 0.2).astype(np.float32)
    if kind == "fullrows":
        m[0] = 1.0
        if Bm > 2:
            m[2] = 1.0
    return m


# (B, H, Lq, Lk, dh, Bm): dh in {1, 4, 5, 32, 64, 128}, lengths at 1 and at the 64-row tile edges +-1, 257, Lq != Lk,
# H in {1, 2, 8}, Bm = B (the Transformer's masks), 1 and 3 (dividing H*B)
CASES = [
    (2, 1, 1, 1, 1, 2), (3, 2, 63, 63, 4, 3), (2, 2, 64, 64, 5, 2), (2, 8, 65, 65, 32, 2), (1, 2, 127, 129, 64, 1),
    (1, 1, 128, 128, 128, 1), (2, 2, 129, 1, 4, 2), (1, 1, 257, 257, 32, 1), (3, 8, 20, 33, 8, 3),
    (2, 1, 1, 65, 16, 2), (4, 2, 40, 40, 64, 8), (1, 8, 33, 17, 128, 8),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B{}H{}Lq{}Lk{}dh{}Bm{}".format(*c))
@pytest.mark.parametrize("mask_kind", ["none", "pad", "fullrows"])
@pytest.mark.parametrize("causal", [False, True])
def test_attention_matches_oracle(case, mask_kind, causal):
    B, H, Lq, Lk, dh, Bm = case
    if causal and Lq != Lk:
        pytest.skip("causal masking needs Lq == Lk")
    rng = np.random.default_rng(zlib.crc32(repr((case, mask_kind, causal)).encode()))
    q, k, v, g = (rng.standard_normal((B, L, H * dh)).astype(np.float32) for L in (Lq, Lk, Lk, Lq))
    mask = _mask(rng, mask_kind, B, H, Lk, Bm)
    o, lse = attn_fwd(_dev(q), _dev(k), _dev(v), _dev(mask), H, causal)
    ref = O.attention(q, k, v, mask, H, causal)
    oa, gqa, gka, gva = _abs_terms(q, k, v, g, mask, H, causal, 0.0, 0)
    _close(o.cpu().numpy(), ref, oa, "out")
    gq, gk, gv = attn_bwd(_dev(q), _dev(k), _dev(v), _dev(mask), o, lse, _dev(g), H, causal)
    rq, rk, rv = O.attention_grad(q, k, v, g, mask, H, causal)
    _close(gq.cpu().numpy(), rq, gqa, "gq")
    _close(gk.cpu().numpy(), rk, gka, "gk")
    _close(gv.cpu().numpy(), rv, gva, "gv")


def test_fully_padded_row_is_uniform_and_causal_row0_spans_all_keys():
    rng = np.random.default_rng(5)
    B, H, L, dh = 2, 2, 70, 8
    q, k, v = (rng.standard_normal((B, L, H * dh)).astype(np.float32) for _ in range(3))
    mask = np.zeros((B, L), np.float32)
    mask[0] = 1.0                      # example 0: every key is padding
    mask[1, 0] = 1.0                   # example 1: key 0 is padding
    o, _ = attn_fwd(_dev(q), _dev(k), _dev(v), _dev(mask), H, False)
    np.testing.assert_allclose(o.cpu().numpy()[0], np.broadcast_to(v[0].mean(0), (L, H * dh)), rtol=1e-5, atol=1e-6)
    oc, _ = attn_fwd(_dev(q), _dev(k), _dev(v), _dev(mask), H, True)
    np.testing.assert_allclose(oc.cpu().numpy()[1, 0], v[1].mean(0), rtol=1e-5, atol=1e-6)


def test_attention_bit_identical_across_runs():
    rng = np.random.default_rng(9)
    B, H, L, dh = 3, 4, 150, 32
    q, k, v, g = (_dev(rng.standard_normal((B, L, H * dh)).astype(np.float32)) for _ in range(4))
    mask = _dev((rng.random((B, L)) < 0.3).astype(np.float32))
    for rate in (0.0, 0.25):
        o1, l1 = attn_fwd(q, k, v, mask, H, True, rate, 77)
        o2, l2 = attn_fwd(q, k, v, mask, H, True, rate, 77)
        assert torch.equal(o1, o2) and torch.equal(l1, l2)
        b1 = attn_bwd(q, k, v, mask, o1, l1, g, H, True, rate, 77)
        b2 = attn_bwd(q, k, v, mask, o1, l1, g, H, True, rate, 77)
        assert all(torch.equal(x, y) for x, y in zip(b1, b2))


def test_dropout_mask_fraction_and_oracle():
    rng = np.random.default_rng(3)
    B, H, L, dh, rate, seed = 4, 2, 128, 128, 0.3, 0x1234_5678_9ABC_DEF0
    q, k, g = (rng.standard_normal((B, L, H * dh)).astype(np.float32) for _ in range(3))
    v = np.tile(np.eye(L, dtype=np.float32), (B, 1, H)).reshape(B, L, H * dh)   # out[i, j] = dropped p_ij
    o, lse = attn_fwd(_dev(q), _dev(k), _dev(v), None, H, False, rate, seed)
    kept = O.split_heads(o.cpu().numpy(), H) > 0
    keep = O.keep_mask(seed, rate, H * B, L, L)
    assert np.array_equal(kept, keep)
    n = keep.size
    assert abs(keep.sum() - n * (1 - rate)) < 5 * np.sqrt(n * rate * (1 - rate))
    ref = O.attention(q, k, v, None, H, False, rate, seed)
    oa, gqa, gka, gva = _abs_terms(q, k, v, g, None, H, False, rate, seed)
    _close(o.cpu().numpy(), ref, oa, "out")
    gq, gk, gv = attn_bwd(_dev(q), _dev(k), _dev(v), None, o, lse, _dev(g), H, False, rate, seed)
    rq, rk, rv = O.attention_grad(q, k, v, g, None, H, False, rate, seed)
    _close(gq.cpu().numpy(), rq, gqa, "gq")
    _close(gk.cpu().numpy(), rk, gka, "gk")
    _close(gv.cpu().numpy(), rv, gva, "gv")


def test_rate_zero_is_the_no_dropout_path():
    rng = np.random.default_rng(4)
    q, k, v = (_dev(rng.standard_normal((2, 50, 16)).astype(np.float32)) for _ in range(3))
    o1, l1 = attn_fwd(q, k, v, None, 2, False, 0.0, 1)
    o2, l2 = attn_fwd(q, k, v, None, 2, False, 0.0, 987654321)
    assert torch.equal(o1, o2) and torch.equal(l1, l2)


@pytest.mark.parametrize("N,C", [(1, 1), (7, 8), (300, 33), (65, 512)])
@pytest.mark.parametrize("residual", [False, True])
def test_add_layernorm_matches_oracle(N, C, residual):
    rng = np.random.default_rng(N * 1000 + C)
    x = rng.standard_normal((N, C)).astype(np.float32)
    r = rng.standard_normal((N, C)).astype(np.float32) if residual else None
    gamma, beta = rng.standard_normal(C).astype(np.float32), rng.standard_normal(C).astype(np.float32)
    gy = rng.standard_normal((N, C)).astype(np.float32)
    yf, y = _guarded(N * C)
    lib = _lib()
    dx, dr, dg, db, dgy = (_dev(a) for a in (x, r, gamma, beta, gy))      # alive until the kernels have run
    assert lib.dr_add_layernorm_fwd(dx.data_ptr(), None if dr is None else dr.data_ptr(), dg.data_ptr(),
                                    db.data_ptr(), N, C, 1e-8, y.data_ptr(), _stream()) == 0
    bufs = [_guarded(N * C), _guarded(C), _guarded(C)]
    assert lib.dr_add_layernorm_bwd(dx.data_ptr(), None if dr is None else dr.data_ptr(), dg.data_ptr(),
                                    dgy.data_ptr(), N, C, 1e-8, *(b[1].data_ptr() for b in bufs), _stream()) == 0
    torch.cuda.synchronize()
    _check_guards(yf, N * C)
    for full, t in bufs:
        _check_guards(full, t.numel())
    ref = O.layer_norm(x, r, gamma, beta)
    s = x.astype(np.float64) + (0 if r is None else r)
    sd = np.sqrt(((s - s.mean(-1, keepdims=True)) ** 2).mean(-1, keepdims=True) + 1e-8)
    na = (np.abs(s) + np.abs(s).mean(-1, keepdims=True)) / sd * 4
    _close(y.cpu().numpy().reshape(N, C), ref, np.abs(gamma) * na + np.abs(beta), "y")
    gx, gg, gb = O.layer_norm_grad(x, r, gamma, gy)
    ga = np.abs(gy) * np.abs(gamma)
    gxa = (ga + ga.mean(-1, keepdims=True) + na * (ga * na).mean(-1, keepdims=True)) / sd * 4
    _close(bufs[0][1].cpu().numpy().reshape(N, C), gx, gxa, "gx")
    _close(bufs[1][1].cpu().numpy(), gg, (np.abs(gy) * na).sum(0), "ggamma")
    _close(bufs[2][1].cpu().numpy(), gb, np.abs(gy).sum(0), "gbeta")


@pytest.mark.parametrize("N,V", [(1, 1), (9, 2), (130, 50), (33, 5000)])
def test_softmax_rows_matches_oracle(N, V):
    rng = np.random.default_rng(N + V)
    x = (rng.standard_normal((N, V)) * 3).astype(np.float32)
    gy = rng.standard_normal((N, V)).astype(np.float32)
    yf, y = _guarded(N * V)
    gf, gx = _guarded(N * V)
    lib = _lib()
    dx, dgy = _dev(x), _dev(gy)
    assert lib.dr_softmax_rows_fwd(dx.data_ptr(), N, V, y.data_ptr(), _stream()) == 0
    assert lib.dr_softmax_rows_bwd(y.data_ptr(), dgy.data_ptr(), N, V, gx.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    _check_guards(yf, N * V)
    _check_guards(gf, N * V)
    ref = O.softmax(x.astype(np.float64))
    _close(y.cpu().numpy().reshape(N, V), ref, ref * (1 + np.abs(x) + np.abs(x).max(-1, keepdims=True)) * 4, "y")
    yg = y.cpu().numpy().reshape(N, V)
    ga = np.abs(yg) * (np.abs(gy) + (np.abs(gy) * np.abs(yg)).sum(-1, keepdims=True))
    _close(gx.cpu().numpy().reshape(N, V), O.softmax_grad(yg, gy), ga, "gx")


# ---- layers ---------------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().cpu().numpy()


def test_multi_head_attention_layer_and_autograd():
    from deep_recommenders.keras.models.nlp import MultiHeadAttention
    rng = np.random.default_rng(11)
    B, L, S, d = 3, 10, 7, 12
    x = torch.from_numpy(rng.standard_normal((B, L, d)).astype(np.float32)).cuda().requires_grad_()
    kv = torch.from_numpy(rng.standard_normal((B, S, d)).astype(np.float32)).cuda().requires_grad_()
    masks = torch.from_numpy(rng.random((B, S)) < 0.3).cuda()
    layer = MultiHeadAttention(3, 4, dropout_rate=0.5, seed=1)
    layer.eval()
    out = layer([x, kv, kv, masks])
    wq, wk, wv = (_np(w).astype(np.float64) for w in (layer._weights_queries, layer._weights_keys,
                                                      layer._weights_values))
    xn, kn = _np(x).astype(np.float64), _np(kv).astype(np.float64)
    ref = O.attention(xn @ wq, kn @ wk, kn @ wv, masks.cpu().numpy().astype(np.float32), 3, False)
    np.testing.assert_allclose(_np(out), ref, rtol=1e-4, atol=2e-5)
    g = rng.standard_normal(out.shape).astype(np.float32)
    out.backward(torch.from_numpy(g).cuda())
    gq, gk, gv = O.attention_grad(xn @ wq, kn @ wk, kn @ wv, g, masks.cpu().numpy().astype(np.float32), 3)
    np.testing.assert_allclose(_np(layer._weights_queries.grad), xn.reshape(-1, d).T @ gq.reshape(-1, 12),
                               rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(_np(x.grad), gq @ wq.T, rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(_np(kv.grad), gk @ wk.T + gv @ wv.T, rtol=1e-3, atol=1e-4)
    layer.train()                       # dropout only in training mode
    assert not torch.equal(layer([x, kv, kv, masks]), out)
    layer.eval()
    assert torch.equal(layer([x, kv, kv, masks]), out)


def _transformer_weights(t):
    w = {"embeddings": _np(t.embeddings)}
    for pre, mods in (("enc_mha", t.EncoderMultiHeadAttentions), ("dec_mha0", t.DecoderMultiHeadAttentions0),
                      ("dec_mha1", t.DecoderMultiHeadAttentions1)):
        for i, m in enumerate(mods):
            w[f"{pre}{i}_wq"], w[f"{pre}{i}_wk"], w[f"{pre}{i}_wv"] = (
                _np(m._weights_queries), _np(m._weights_keys), _np(m._weights_values))
    for pre, mods in (("enc_ln0", t.EncoderLayerNorms0), ("enc_ln1", t.EncoderLayerNorms1),
                      ("dec_ln0", t.DecoderLayerNorms0), ("dec_ln1", t.DecoderLayerNorms1),
                      ("dec_ln2", t.DecoderLayerNorms2)):
        for i, m in enumerate(mods):
            w[f"{pre}{i}_gamma"], w[f"{pre}{i}_beta"] = _np(m.gamma), _np(m.beta)
    for pre, mods in (("enc_ff", t.EncoderPositionWiseFeedForwards), ("dec_ff", t.DecoderPositionWiseFeedForwards)):
        for i, m in enumerate(mods):
            w[f"{pre}{i}_wi"], w[f"{pre}{i}_bi"] = _np(m.weights_inner), _np(m.bias_inner)
            w[f"{pre}{i}_wo"], w[f"{pre}{i}_bo"] = _np(m.weights_out), _np(m.bias_out)
    return w


def test_transformer_matches_oracle():
    from deep_recommenders.keras.models.nlp import Transformer
    rng = np.random.default_rng(21)
    t = Transformer(50, 8, n_heads=2, encoder_stack=2, decoder_stack=2, feed_forward_size=16, dropout_rate=0.0,
                    seed=3)
    enc = rng.integers(0, 50, size=(4, 12))
    dec = rng.integers(0, 50, size=(4, 12))
    enc[0, 5:] = 0
    dec[1, :3] = 0
    t.eval()
    out = t(torch.from_numpy(enc).cuda(), torch.from_numpy(dec).cuda())
    assert out.shape == (4, 12, 50)
    ref = O.transformer(_transformer_weights(t), enc, dec, 2)
    np.testing.assert_allclose(_np(out), ref, rtol=1e-4, atol=1e-6)
    out.log().sum().backward()
    assert t.embeddings.grad is not None and torch.isfinite(t.embeddings.grad).all()


def test_layers_match_golden():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "nlp_golden.npz"))
    from deep_recommenders.keras.models.nlp import multi_head_attention as mha_mod, transformer as tr
    for key in [k[:-4] for k in g.files if k.startswith("f32_sdpa_") and k.endswith("_out")]:
        masking, future = bool(g[key + "_masking"]), bool(g[key + "_future"])
        layer = mha_mod.ScaledDotProductAttention(masking=masking, future=future)
        ins = [torch.from_numpy(g[key + n]).cuda() for n in ("_q", "_k", "_v")]
        if masking:
            ins.append(torch.from_numpy(g[key + "_mask"]).cuda())
        np.testing.assert_allclose(_np(layer(ins)), g[key + "_out"], rtol=1e-4, atol=1e-6, err_msg=key)
    for key in [k[:-4] for k in g.files if k.startswith("f32_mha_") and k.endswith("_out")]:
        H, dh = int(g[key + "_heads"]), int(g[key + "_head_dim"])
        masking, future = bool(g[key + "_masking"]), bool(g[key + "_future"])
        layer = mha_mod.MultiHeadAttention(H, dh, dropout_rate=0.0, masking=masking, future=future)
        ins = [torch.from_numpy(g[key + n]).cuda() for n in ("_q", "_k", "_v")]
        if masking:
            ins.append(torch.from_numpy(g[key + "_mask"]).cuda())
        layer(ins)
        with torch.no_grad():
            for name in ("queries", "keys", "values"):
                getattr(layer, "_weights_" + name).copy_(torch.from_numpy(g[key + "_w" + name[0]]))
        np.testing.assert_allclose(_np(layer(ins)), g[key + "_out"], rtol=1e-4, atol=1e-6, err_msg=key)
    x = torch.from_numpy(g["f32_ln_x"]).cuda()
    ln = tr.LayerNormalization()
    ln(x)
    with torch.no_grad():
        ln.gamma.copy_(torch.from_numpy(g["f32_ln_gamma"]))
        ln.beta.copy_(torch.from_numpy(g["f32_ln_beta"]))
    np.testing.assert_allclose(_np(ln(x)), g["f32_ln_out"], rtol=1e-5, atol=1e-5)
    pe = tr.PositionEncoding(int(g["f32_pe_dim"]))(torch.zeros(tuple(g["f32_pe_shape"])).cuda())
    np.testing.assert_array_equal(_np(pe), g["f32_pe_out"])


def test_transformer_matches_golden():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "nlp_golden.npz"))
    from deep_recommenders.keras.models.nlp import Transformer
    t = Transformer(50, 8, n_heads=2, encoder_stack=2, decoder_stack=2, feed_forward_size=16, dropout_rate=0.0)
    enc, dec = g["f32_tr_enc"], g["f32_tr_dec"]
    t.eval()
    t(torch.from_numpy(enc).cuda(), torch.from_numpy(dec).cuda())
    w = {k[len("f32_tr_w_"):]: g[k] for k in g.files if k.startswith("f32_tr_w_")}
    _load_transformer_weights(t, w)
    out = t(torch.from_numpy(enc).cuda(), torch.from_numpy(dec).cuda())
    np.testing.assert_allclose(_np(out), g["f32_tr_out"], rtol=1e-4, atol=1e-6)


def _load_transformer_weights(t, w):
    mine = _transformer_weights(t)
    params = {"embeddings": t.embeddings}
    for pre, mods in (("enc_mha", t.EncoderMultiHeadAttentions), ("dec_mha0", t.DecoderMultiHeadAttentions0),
                      ("dec_mha1", t.DecoderMultiHeadAttentions1)):
        for i, m in enumerate(mods):
            params.update({f"{pre}{i}_wq": m._weights_queries, f"{pre}{i}_wk": m._weights_keys,
                           f"{pre}{i}_wv": m._weights_values})
    for pre, mods in (("enc_ln0", t.EncoderLayerNorms0), ("enc_ln1", t.EncoderLayerNorms1),
                      ("dec_ln0", t.DecoderLayerNorms0), ("dec_ln1", t.DecoderLayerNorms1),
                      ("dec_ln2", t.DecoderLayerNorms2)):
        for i, m in enumerate(mods):
            params.update({f"{pre}{i}_gamma": m.gamma, f"{pre}{i}_beta": m.beta})
    for pre, mods in (("enc_ff", t.EncoderPositionWiseFeedForwards), ("dec_ff", t.DecoderPositionWiseFeedForwards)):
        for i, m in enumerate(mods):
            params.update({f"{pre}{i}_wi": m.weights_inner, f"{pre}{i}_bi": m.bias_inner,
                           f"{pre}{i}_wo": m.weights_out, f"{pre}{i}_bo": m.bias_out})
    assert set(params) == set(mine) == set(w)
    with torch.no_grad():
        for k, p in params.items():
            p.copy_(torch.from_numpy(np.asarray(w[k], np.float32)))


# ---- the reference's test_save_model and the example's model --------------------------------------------------------
def _classifier(units=1, act="sigmoid", **kw):
    from deep_recommenders.keras.layers import Dense, Model
    from deep_recommenders.keras.models.nlp import Transformer

    class Classifier(Model):
        def __init__(self, vocab_size, model_dim, n_heads, encoder_stack, decoder_stack, feed_forward_size,
                     dropout_rate=0.1, seed=None):
            super().__init__()
            self.transformer = Transformer(vocab_size, model_dim, n_heads=n_heads, encoder_stack=encoder_stack,
                                           decoder_stack=decoder_stack, feed_forward_size=feed_forward_size,
                                           dropout_rate=dropout_rate, seed=seed)
            self.head = Dense(units, activation=act, seed=seed)
            self.built = True

        def call(self, inputs, **kwargs):
            enc, dec = inputs
            return self.head(self.transformer(enc, dec).mean(dim=1))   # GlobalAveragePooling1D

        def get_config(self):
            return {**super().get_config(), "transformer": self.transformer.get_config(),
                    "head": self.head.get_config()}

    return Classifier(**kw)


def test_reference_save_model():
    """tests/keras/test_transformer.py: Transformer(5000, 8, 2, 2 + 2, ff 50) on [10, 256] ids, pooled, Dense(1,
    sigmoid); predict, save, load, equal configs and predictions."""
    rng = np.random.default_rng(0)
    cfg = dict(vocab_size=5000, model_dim=8, n_heads=2, encoder_stack=2, decoder_stack=2, feed_forward_size=50)
    model = _classifier(**cfg, seed=1)
    enc = torch.from_numpy(rng.integers(0, 5000, size=(10, 256))).cuda()
    dec = torch.from_numpy(rng.integers(0, 5000, size=(10, 256))).cuda()
    pred = model.predict([enc, dec])
    assert pred.shape == (10, 1)
    assert torch.equal(model.predict([enc, dec]), pred)      # dropout is off in predict
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "transformer_model")
        model.save(path)
        blob = torch.load(path, weights_only=False)
        loaded = _classifier(**cfg)
        loaded.predict([enc, dec])
        loaded.load_state_dict(blob["state"])
        assert loaded.get_config() == model.get_config() == blob["config"]
        assert loaded.transformer.get_config() == model.transformer.get_config()
        assert torch.equal(loaded.predict([enc, dec]), pred)


def test_example_model_fit_lowers_loss():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples"))
    import train_transformer_on_synthetic_keras as ex
    hist = ex.train_model(vocab_size=200, max_len=24, batch_size=64, epochs=4, steps_per_epoch=25, seed=0)
    print("losses by epoch", hist["loss"])
    assert hist["loss"][-1] < hist["loss"][0]
