"""Generates tests/golden/nlp_golden.npz by EXECUTING THE REFERENCE'S OWN keras/models/nlp/multi_head_attention.py and
transformer.py (read from a checkout of the reference, never copied) under the numpy-backed `tensorflow` stand-in in
oracle/tf_shim.  Nothing calls this script: the .npz file is committed and the tests read only it.  Run it by hand, on
any machine (no GPU needed):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_nlp_golden.py

The stand-in lacks ops these files use; this script adds them for its own process only (TensorFlow's documented
semantics, computed in the inputs' dtype), so the shim files and the other golden vectors are untouched:
  tensorflow.keras.backend (dtype, cast, gather, batch_dot, dot, transpose, softmax, relu, tile, expand_dims, shape,
  equal, minimum, and dropout as the identity -- the rate-0 / inference form), tensorflow.keras.layers and
  tensorflow.keras.callbacks as importable modules, tf.split, tf.linalg.LinearOperatorLowerTriangular, tf.nn.moments,
  Layer.add_weight with the glorot_uniform / uniform / zero / one initializers, and a Layer.__call__ that passes the
  shapes of a list input to build.
It writes only tests/golden/nlp_golden.npz: for each dtype (prefix f32_ / f64_)
  sdpa_<case>_{q,k,v,mask,masking,future,out}   ScaledDotProductAttention with masking / future combinations,
                                                        fully padded rows, Lq != Lk cross-attention, Bm < batch
  mha_<case>_{q,k,v,mask,wq,wk,wv,heads,head_dim,masking,future,out}   MultiHeadAttention (dropout 0)
  ln_{x,gamma,beta,out}                                 LayerNormalization
  pe_{dim,shape,out}                                    PositionEncoding
  tr_{enc,dec,out}, tr_w_<name>                         Transformer(50, 8, 2 heads, 2 + 2 stacks, ff 16), dropout 0
  tr_config_keys
ScaledDotProductAttention casts its inputs to float32 (:68-70), so the f64_ attention outputs are float32 results of
float64 inputs (MultiHeadAttention's projections are float64 there).
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_nlp_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"

_RNG = np.random.RandomState(29)


def _extend_shim():
    T = tf.convert_to_tensor
    a = np.asarray
    dt = {"float32": np.float32, "float64": np.float64, "int32": np.int32, "int64": np.int64}

    def softmax(x, axis=-1):
        x = a(x)
        e = np.exp(x - x.max(axis, keepdims=True))
        return T(e / e.sum(axis, keepdims=True))

    K = types.ModuleType("tensorflow.keras.backend")
    K.dtype = lambda x: a(x).dtype.name
    K.cast = lambda x, d: T(a(x).astype(dt[d]))
    K.gather = lambda p, i: T(a(p)[a(i)])
    K.batch_dot = lambda x, y: T(np.matmul(a(x), a(y)))
    K.dot = lambda x, y: T(np.matmul(a(x), a(y)))
    K.transpose = lambda x: T(a(x).T)
    K.softmax = softmax
    K.relu = lambda x: T(np.maximum(a(x), 0))
    K.tile = lambda x, n: T(np.tile(a(x), n))
    K.expand_dims = lambda x, axis=-1: T(np.expand_dims(a(x), axis))
    K.shape = lambda x: a(a(x).shape)
    K.equal = lambda x, y: T(a(x) == a(y))
    K.minimum = lambda x, y: np.minimum(x, y)
    K.dropout = lambda x, level, **kw: x
    layers_mod = types.ModuleType("tensorflow.keras.layers")
    layers_mod.__dict__.update(vars(tf.keras.layers))
    cb_mod = types.ModuleType("tensorflow.keras.callbacks")
    cb_mod.Callback = type("Callback", (), {"__init__": lambda self: None})
    keras_mod = types.ModuleType("tensorflow.keras")
    keras_mod.__dict__.update(vars(tf.keras))
    keras_mod.backend, keras_mod.layers, keras_mod.callbacks = K, layers_mod, cb_mod
    sys.modules.update({"tensorflow.keras": keras_mod, "tensorflow.keras.backend": K,
                        "tensorflow.keras.layers": layers_mod, "tensorflow.keras.callbacks": cb_mod})
    tf.keras = keras_mod
    tf.split = lambda x, n, axis=0: [T(p) for p in np.split(a(x), n, axis=axis)]
    tf.linalg = types.SimpleNamespace(LinearOperatorLowerTriangular=lambda m: types.SimpleNamespace(
        to_dense=lambda: T(np.tril(a(m)))))
    tf.nn.moments = lambda x, axes, keepdims=False: (
        T(a(x).mean(tuple(axes), keepdims=keepdims)),
        T(((a(x) - a(x).mean(tuple(axes), keepdims=True)) ** 2).mean(tuple(axes), keepdims=keepdims)))

    def add_weight(self, shape=None, initializer=None, name=None, trainable=True, **k):
        d = tf.DEFAULT_DTYPE[0]
        shape = tuple(int(s) for s in shape)
        if initializer == "glorot_uniform":
            lim = np.sqrt(6.0 / (shape[0] + shape[-1]))
            return _RNG.uniform(-lim, lim, size=shape).astype(d)
        if initializer == "uniform":
            return _RNG.uniform(-0.05, 0.05, size=shape).astype(d)
        return (np.zeros if initializer == "zero" else np.ones)(shape, d)

    def call(self, *args, **kwargs):
        if not self.built:
            first = args[0]
            shp = [tuple(a(x).shape) for x in first] if isinstance(first, (list, tuple)) else a(first).shape
            self.build(shp)
            self.built = True
        return self.call(*args, **kwargs)

    tf.keras.layers.Layer.add_weight = add_weight
    tf.keras.layers.Layer.__call__ = call


def generate(dtype, out):
    from deep_recommenders.keras.models.nlp import multi_head_attention as M
    from deep_recommenders.keras.models.nlp import transformer as T
    tf.set_default_dtype(dtype)
    pre = "f32_" if dtype == np.float32 else "f64_"
    rng = np.random.RandomState(17)

    def mask_for(Bm, Lk, full=()):
        m = (rng.random_sample((Bm, Lk)) < 0.25).astype(np.float32)
        for r in full:
            m[r] = 1.0
        return m

    # (tag, B, Lq, Lk, d, masking, future, Bm, fully padded mask rows)
    for tag, B, Lq, Lk, d, masking, future, Bm, full in [
            ("plain", 3, 5, 5, 4, False, False, 3, ()),
            ("mask", 3, 6, 6, 4, True, False, 3, ()),
            ("future", 2, 6, 6, 5, False, True, 2, ()),
            ("mask_future", 4, 7, 7, 4, True, True, 4, ()),
            ("padded_rows", 3, 5, 5, 3, True, False, 3, (1,)),
            ("causal_key0", 2, 6, 6, 4, True, True, 2, ()),
            ("cross", 2, 4, 9, 6, True, False, 2, ()),
            ("bm_lt_b", 6, 5, 8, 4, True, False, 2, ())]:
        q, k, v = (rng.standard_normal((B, L, d)).astype(dtype) for L in (Lq, Lk, Lk))
        m = mask_for(Bm, Lk, full)
        if tag == "causal_key0":
            m[:, 0] = 1.0
        layer = M.ScaledDotProductAttention(masking=masking, future=future)
        res = layer([q, k, v, m] if masking else [q, k, v])
        key = f"{pre}sdpa_{tag}"
        out.update({key + "_q": q, key + "_k": k, key + "_v": v, key + "_mask": m, key + "_masking": masking,
                    key + "_future": future, key + "_out": np.asarray(res, dtype)})

    # (tag, B, Lq, Lk, d_in, heads, head_dim, masking, future)
    for tag, B, Lq, Lk, d_in, H, dh, masking, future in [
            ("self_mask", 3, 6, 6, 8, 2, 4, True, False),
            ("self_mask_future", 2, 7, 7, 6, 3, 2, True, True),
            ("cross_nomask", 2, 5, 8, 5, 2, 3, False, False),
            ("self_future_nomask", 2, 5, 5, 4, 4, 1, False, True)]:
        q = rng.standard_normal((B, Lq, d_in)).astype(dtype)
        k = rng.standard_normal((B, Lk, d_in)).astype(dtype)
        v = rng.standard_normal((B, Lk, d_in)).astype(dtype)
        m = mask_for(B, Lk, (0,) if masking else ())
        layer = M.MultiHeadAttention(H, dh, dropout_rate=0.0, masking=masking, future=future)
        res = layer([q, k, v, m] if masking else [q, k, v])
        key = f"{pre}mha_{tag}"
        out.update({key + "_q": q, key + "_k": k, key + "_v": v, key + "_mask": m, key + "_heads": H,
                    key + "_head_dim": dh, key + "_masking": masking, key + "_future": future,
                    key + "_wq": np.asarray(layer._weights_queries, dtype),
                    key + "_wk": np.asarray(layer._weights_keys, dtype),
                    key + "_wv": np.asarray(layer._weights_values, dtype),
                    key + "_out": np.asarray(res, dtype)})

    x = (rng.standard_normal((4, 3, 10)) * 2 + 1).astype(dtype)
    ln = T.LayerNormalization()
    ln(x)
    ln.gamma = rng.standard_normal(10).astype(dtype)
    ln.beta = rng.standard_normal(10).astype(dtype)
    out.update({pre + "ln_x": x, pre + "ln_gamma": ln.gamma, pre + "ln_beta": ln.beta,
                pre + "ln_out": np.asarray(ln(x), dtype)})
    pe_shape = (2, 13, 6)
    out.update({pre + "pe_dim": 6, pre + "pe_shape": np.asarray(pe_shape),
                pre + "pe_out": np.asarray(T.PositionEncoding(6)(np.zeros(pe_shape, dtype)))})

    tr = T.Transformer(50, 8, n_heads=2, encoder_stack=2, decoder_stack=2, feed_forward_size=16, dropout_rate=0.0)
    enc = rng.randint(0, 50, size=(3, 12))
    dec = rng.randint(0, 50, size=(3, 12))
    enc[0, 7:] = 0
    dec[1, :4] = 0
    tr.build(None)
    w = {"embeddings": tr.embeddings}
    for p, mods in (("enc_mha", tr.EncoderMultiHeadAttentions), ("dec_mha0", tr.DecoderMultiHeadAttentions0),
                    ("dec_mha1", tr.DecoderMultiHeadAttentions1)):
        for i, m in enumerate(mods):
            m.build([(None, None, 8)] * 3)
            m.built = True
            w.update({f"{p}{i}_wq": m._weights_queries, f"{p}{i}_wk": m._weights_keys, f"{p}{i}_wv": m._weights_values})
    for p, mods in (("enc_ln0", tr.EncoderLayerNorms0), ("enc_ln1", tr.EncoderLayerNorms1),
                    ("dec_ln0", tr.DecoderLayerNorms0), ("dec_ln1", tr.DecoderLayerNorms1),
                    ("dec_ln2", tr.DecoderLayerNorms2)):
        for i, m in enumerate(mods):
            m.build((None, None, 8))
            m.built = True
            m.gamma = (1 + 0.3 * rng.standard_normal(8)).astype(dtype)      # not the identity initialisation
            m.beta = (0.2 * rng.standard_normal(8)).astype(dtype)
            w.update({f"{p}{i}_gamma": m.gamma, f"{p}{i}_beta": m.beta})
    for p, mods in (("enc_ff", tr.EncoderPositionWiseFeedForwards), ("dec_ff", tr.DecoderPositionWiseFeedForwards)):
        for i, m in enumerate(mods):
            m.build((None, None, 8))
            m.built = True
            w.update({f"{p}{i}_wi": m.weights_inner, f"{p}{i}_bi": m.bias_inner, f"{p}{i}_wo": m.weights_out,
                      f"{p}{i}_bo": m.bias_out})
    tr.built = True
    res = tr(enc, dec)
    out.update({pre + "tr_enc": enc.astype(np.int64), pre + "tr_dec": dec.astype(np.int64),
                pre + "tr_out": np.asarray(res, dtype)})
    out.update({f"{pre}tr_w_{k}": np.asarray(v, dtype) for k, v in w.items()})
    out[pre + "tr_config_keys"] = np.asarray(sorted(k for k in tr.get_config() if k != "name"))


if __name__ == "__main__":
    _extend_shim()
    out = {}
    for d in (np.float32, np.float64):
        generate(d, out)
    path = os.path.join(HERE, "nlp_golden.npz")
    np.savez(path, **out)
    print(f"wrote {path}: {len(out)} arrays")
