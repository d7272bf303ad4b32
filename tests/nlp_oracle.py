"""numpy restatement of the Transformer pieces (keras/models/nlp in the reference) in float64 or float32: the fused
attention with its padding constant, causal rule and dropout hash, LayerNorm of a sum, the row softmax, the sinusoid
position encoding and a whole Transformer forward; plus the float64 closed-form gradients of the attention, the
LayerNorm and the softmax.

In float64 a score the padding constant was added to is rounded to float32, as the reference's float32 add does:
fl32(s - 4294967296) is exactly -4294967296 for |s| < 256, which is what makes a fully padded row uniform."""
import numpy as np

NEG = np.float32(-4294967296.0)
_M64 = (1 << 64) - 1


def keep_mask(seed, rate, R, Lq, Lk):
    """keep(r, i, j) of dr_mha_attn_fwd as a bool array [R, Lq, Lk] (the splitmix64 finalizer in the header)."""
    c = np.arange(R * Lq * Lk, dtype=np.uint64).reshape(R, Lq, Lk)
    with np.errstate(over="ignore"):
        z = np.uint64(int(seed) & _M64) + (c + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    thr = np.uint64(int(float(np.float32(rate)) * 16777216.0))
    return (z >> np.uint64(40)) >= thr


def keep_scale(rate):
    return np.float32(1.0) / (np.float32(1.0) - np.float32(rate))


def split_heads(x, H):
    """[B, L, H*dh] -> [H*B, L, dh], row r = h*B + b (concat(split(x, H, axis=2), axis=0))."""
    B, L, HD = x.shape
    return x.reshape(B, L, H, HD // H).transpose(2, 0, 1, 3).reshape(H * B, L, HD // H)


def merge_heads(x, H):
    HB, L, dh = x.shape
    return x.reshape(H, HB // H, L, dh).transpose(1, 2, 0, 3).reshape(HB // H, L, H * dh)


def scores(q, k, mask, causal, dtype=np.float64):
    """(s [R, Lq, Lk], replaced [R, Lq, Lk] or None) for split heads q [R, Lq, dh], k [R, Lk, dh]."""
    q, k = q.astype(dtype), k.astype(dtype)
    dh = q.shape[-1]
    div = dtype(np.float32(np.sqrt(dh)))
    s = np.einsum("rid,rjd->rij", q, k) / div
    if mask is not None:
        R, Bm = q.shape[0], mask.shape[0]
        m = np.tile(np.asarray(mask, np.float32), (R // Bm, 1))[:, None, :]
        add = (m * NEG).astype(np.float32)
        if dtype == np.float32:
            s = s + add
        else:
            s = np.where(add != 0, (s.astype(np.float32) + add).astype(np.float64), s)
    rep = None
    if causal:
        Lq, Lk = s.shape[1:]
        rep = np.broadcast_to(np.triu(np.ones((Lq, Lk), bool), 1), s.shape)
        s = np.where(rep, dtype(NEG), s)
    return s, rep


def softmax(s):
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def attention(q, k, v, mask=None, H=1, causal=False, rate=0.0, seed=0, dtype=np.float64):
    """out [B, Lq, H*dh] of dr_mha_attn_fwd (q, k, v in the projections' layout)."""
    qs, ks, vs = (split_heads(np.asarray(x, dtype), H) for x in (q, k, v))
    s, _ = scores(qs, ks, mask, causal, dtype)
    p = softmax(s)
    if rate > 0:
        p = np.where(keep_mask(seed, rate, *s.shape), p * dtype(keep_scale(rate)), dtype(0))
    return merge_heads(np.einsum("rij,rjd->rid", p, vs), H)


def attention_grad(q, k, v, g, mask=None, H=1, causal=False, rate=0.0, seed=0):
    """float64 (gq, gk, gv) of TensorFlow's autodiff of the attention: the mask add passes the gradient, the causal
    where gives 0 at replaced positions."""
    qs, ks, vs, gs = (split_heads(np.asarray(x, np.float64), H) for x in (q, k, v, g))
    s, rep = scores(qs, ks, mask, causal)
    p = softmax(s)
    kp = keep_mask(seed, rate, *s.shape) * np.float64(keep_scale(rate)) if rate > 0 else 1.0
    pd = p * kp
    gv = np.einsum("rij,rid->rjd", pd, gs)
    dpd = np.einsum("rid,rjd->rij", gs, vs)
    dp = dpd * kp
    ds = p * (dp - (p * dp).sum(-1, keepdims=True))
    if rep is not None:
        ds = np.where(rep, 0.0, ds)
    div = np.float64(np.float32(np.sqrt(qs.shape[-1])))
    gq = np.einsum("rij,rjd->rid", ds, ks) / div
    gk = np.einsum("rij,rid->rjd", ds, qs) / div
    return merge_heads(gq, H), merge_heads(gk, H), merge_heads(gv, H)


def layer_norm(x, residual, gamma, beta, eps=1e-8, dtype=np.float64):
    s = np.asarray(x, dtype) + (0 if residual is None else np.asarray(residual, dtype))
    mu = s.mean(-1, keepdims=True)
    var = ((s - mu) ** 2).mean(-1, keepdims=True)
    return np.asarray(gamma, dtype) * ((s - mu) / (var + dtype(eps)) ** dtype(0.5)) + np.asarray(beta, dtype)


def layer_norm_grad(x, residual, gamma, gy, eps=1e-8):
    """float64 (gx, ggamma, gbeta); gx is also the residual's gradient."""
    s = np.asarray(x, np.float64) + (0 if residual is None else np.asarray(residual, np.float64))
    C = s.shape[-1]
    mu = s.mean(-1, keepdims=True)
    den = (((s - mu) ** 2).mean(-1, keepdims=True) + eps) ** 0.5
    n = (s - mu) / den
    gy = np.asarray(gy, np.float64)
    gn = gy * gamma
    gx = (gn - gn.mean(-1, keepdims=True) - n * (gn * n).mean(-1, keepdims=True)) / den
    return gx, (gy * n).reshape(-1, C).sum(0), gy.reshape(-1, C).sum(0)


def softmax_grad(y, gy):
    y, gy = np.asarray(y, np.float64), np.asarray(gy, np.float64)
    return y * (gy - (gy * y).sum(-1, keepdims=True))


def position_encoding(L, d):
    pe = np.zeros((L, d))
    for pos in range(L):
        for i in range(d):
            pe[pos, i] = pos / np.power(10000, (i - i % 2) / d)
    pe[:, 0::2] = np.sin(pe[:, 0::2])
    pe[:, 1::2] = np.cos(pe[:, 1::2])
    return pe


def transformer(w, enc_ids, dec_ids, n_heads, dtype=np.float64):
    """Transformer.call with dropout 0.  `w`: 'embeddings' and per sub-layer '<prefix>{i}_<name>' arrays, prefixes
    enc_mha / enc_ln0 / enc_ff / enc_ln1 / dec_mha0 / dec_ln0 / dec_mha1 / dec_ln1 / dec_ff / dec_ln2; names wq wk wv,
    gamma beta, wi bi wo bo."""
    E = np.asarray(w["embeddings"], dtype)
    d = E.shape[1]
    f = lambda a: np.asarray(a, dtype)

    def embed(ids):
        x = E[ids] * dtype(d ** 0.5)
        return x + position_encoding(ids.shape[1], d).astype(np.float32).astype(dtype)

    def mha(p, x, kv, masks, future):
        q, k, v = x @ f(w[p + "_wq"]), kv @ f(w[p + "_wk"]), kv @ f(w[p + "_wv"])
        return attention(q, k, v, masks, n_heads, future, dtype=dtype)

    def ln(p, x, r):
        return layer_norm(x, r, w[p + "_gamma"], w[p + "_beta"], dtype=dtype)

    def ff(p, x):
        return np.maximum(x @ f(w[p + "_wi"]) + f(w[p + "_bi"]), 0) @ f(w[p + "_wo"]) + f(w[p + "_bo"])

    n_enc = sum(1 for key in w if key.startswith("enc_mha") and key.endswith("_wq"))
    n_dec = sum(1 for key in w if key.startswith("dec_mha0") and key.endswith("_wq"))
    enc_masks = (enc_ids == 0).astype(np.float32)
    x = embed(enc_ids)
    for i in range(n_enc):
        a = ln(f"enc_ln0{i}", mha(f"enc_mha{i}", x, x, enc_masks, False), x)
        x = ln(f"enc_ln1{i}", ff(f"enc_ff{i}", a), a)
    dec_masks = (dec_ids == 0).astype(np.float32)
    y = embed(dec_ids)
    for i in range(n_dec):
        m = ln(f"dec_ln0{i}", mha(f"dec_mha0{i}", y, y, dec_masks, True), y)
        a = ln(f"dec_ln1{i}", mha(f"dec_mha1{i}", m, x, enc_masks, False), m)
        y = ln(f"dec_ln2{i}", ff(f"dec_ff{i}", a), a)
    return softmax(y @ E.T)
