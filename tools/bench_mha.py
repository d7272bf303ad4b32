"""Multi-head self-attention at a sequence-recommender shape, and the whole Transformer step:

  attention    B = 4096, L = 200, H = 8, dh = 32, padding mask (20 % of keys), without and with causal masking:
               CUDA-event times of dr_mha_attn_fwd and of the forward + dr_mha_attn_bwd, against the torch fp32
               composition the reference's form maps to ([H*B, L, L] scores materialised in chunks of --chunk logical
               rows: matmul, scale, mask, where, softmax, matmul, and autograd for the backward; TF32 off), alternating
               in one process.  Useful TFLOP/s are counted in the reference's form, 4*H*B*L*L*dh for the forward and
               twice that for the backward, against the 67 TFLOP/s data-sheet fp32 rate of an H100 SXM.  The largest
               output and gradient differences between the two are reported.
  transformer  the reference example's model (vocab 5000, L 128, B 128, model 8, 2 heads, 2 + 2 stacks, ff 50,
               mean pooled, Dense(2) softmax, categorical cross-entropy, Adam) through the Keras engine, one `fit`
               step per call.  At model_dim 8 every kernel is tiny: this shape measures launch and framework overhead,
               not the kernels.

The card's name and power limit are read in the same run.  Prints one JSON line and writes it to
<--out-dir>/bench_mha.json (default bench_out/, which git ignores).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "examples"))
from bench_dcn_step import card  # noqa: E402
from bench_din import summary, timed  # noqa: E402
from deep_recommenders_b200 import ops  # noqa: E402

FP32_PEAK_TFLOPS = 67.0
NEG = -4294967296.0


def composition(q, k, v, mask, H, causal, chunk, g=None):
    """The reference's ScaledDotProductAttention on split heads, chunk logical rows at a time; with g, also the
    autograd backward.  Returns out (and gq, gk, gv)."""
    B, L, HD = q.shape
    dh = HD // H
    split = lambda x: x.view(B, L, H, dh).permute(2, 0, 1, 3).reshape(H * B, L, dh)
    qs, ks, vs = split(q), split(k), split(v)
    gs = None if g is None else split(g)
    div = float(np.float32(np.sqrt(dh)))
    tri = torch.triu(torch.ones(L, L, dtype=torch.bool, device=q.device), 1)
    outs, grads = [], [[], [], []]
    for r0 in range(0, H * B, chunk):
        r1 = min(H * B, r0 + chunk)
        rows = torch.arange(r0, r1, device=q.device) % B
        a, b, c = (x[r0:r1].detach().requires_grad_(g is not None) for x in (qs, ks, vs))
        with torch.set_grad_enabled(g is not None):
            s = a @ b.transpose(1, 2) / div
            s = s + mask[rows][:, None, :] * NEG
            if causal:
                s = torch.where(tri, torch.full_like(s, NEG), s)
            o = torch.softmax(s, -1) @ c
        outs.append(o.detach())
        if g is not None:
            o.backward(gs[r0:r1])
            for lst, t in zip(grads, (a, b, c)):
                lst.append(t.grad)
    merge = lambda parts: torch.cat(parts).view(H, B, L, dh).permute(1, 2, 0, 3).reshape(B, L, HD)
    if g is None:
        return merge(outs)
    return (merge(outs),) + tuple(merge(p) for p in grads)


def bench_attention(a, causal):
    torch.backends.cuda.matmul.allow_tf32 = False
    gen = torch.Generator(device="cuda").manual_seed(0)
    B, L, H, dh = a.batch, a.seq_len, a.heads, a.head_dim
    q, k, v, g = (torch.randn((B, L, H * dh), device="cuda", generator=gen) for _ in range(4))
    mask = (torch.rand((B, L), device="cuda", generator=gen) < 0.2).float()
    qf, kf, vf = (x.clone().requires_grad_() for x in (q, k, v))

    def fused_fwd():
        return ops.MHAttentionFn.apply(q, k, v, mask, H, causal, 0.0, 0)

    def fused_fwd_bwd():
        out = ops.MHAttentionFn.apply(qf, kf, vf, mask, H, causal, 0.0, 0)
        return torch.autograd.grad(out, (qf, kf, vf), g)

    times = {"fused_fwd": [], "fused_fwd_bwd": [], "torch_fwd": [], "torch_fwd_bwd": []}
    with torch.no_grad():
        fused_fwd(), composition(q, k, v, mask, H, causal, a.chunk)
    for _ in range(a.rounds):              # alternate the two forms so drift hits both alike
        with torch.no_grad():
            times["fused_fwd"] += timed(fused_fwd, a.warmup, a.iters)
            times["torch_fwd"] += timed(lambda: composition(q, k, v, mask, H, causal, a.chunk), 1, a.iters)
        times["fused_fwd_bwd"] += timed(fused_fwd_bwd, a.warmup, a.iters)
        times["torch_fwd_bwd"] += timed(lambda: composition(q, k, v, mask, H, causal, a.chunk, g), 1, a.iters)
    with torch.no_grad():
        out_f = fused_fwd()
    grads_f = fused_fwd_bwd()
    ref = composition(q, k, v, mask, H, causal, a.chunk, g)
    flops = 4.0 * H * B * L * L * dh
    res = {k_: summary(t) for k_, t in times.items()}
    for name, fl in (("fused_fwd", flops), ("fused_fwd_bwd", 3 * flops), ("torch_fwd", flops),
                     ("torch_fwd_bwd", 3 * flops)):
        tf = fl / (res[name]["median_ms"] * 1e-3) / 1e12
        res[name].update(useful_tflops=tf, share_of_fp32_peak=tf / FP32_PEAK_TFLOPS)
    res["speedup_fwd"] = res["torch_fwd"]["median_ms"] / res["fused_fwd"]["median_ms"]
    res["speedup_fwd_bwd"] = res["torch_fwd_bwd"]["median_ms"] / res["fused_fwd_bwd"]["median_ms"]
    res["max_abs_diff"] = {n: float((x - y).abs().max()) for n, x, y in
                           zip(("out", "gq", "gk", "gv"), (out_f,) + tuple(grads_f), ref)}
    res["scores_bytes_per_copy"] = 4 * H * B * L * L
    return res


def bench_transformer(a):
    import train_transformer_on_synthetic_keras as ex
    from deep_recommenders_b200.keras.engine import Adam
    model = ex.TransformerClassifier(5000, 128, seed=0)
    model.compile(optimizer=Adam(beta_1=0.9, beta_2=0.98, epsilon=1e-9), loss="categorical_crossentropy")
    batch = next(ex.synthetic_batches(5000, 128, 128, 0))

    def step():
        model.fit([batch], epochs=1, steps_per_epoch=1)

    ms = timed(step, a.warmup, a.iters * a.rounds)
    s = summary(ms)
    s["examples_per_s"] = 128 / (s["median_ms"] * 1e-3)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--seq-len", type=int, default=200)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--head-dim", type=int, default=32)
    ap.add_argument("--chunk", type=int, default=4096, help="logical rows per chunk of the torch composition")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out-dir", default="bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mha.py needs a CUDA device")
    out = {"card": card(),
           "shape": {"B": a.batch, "L": a.seq_len, "H": a.heads, "dh": a.head_dim, "mask_fraction": 0.2},
           "attention_pad": bench_attention(a, False),
           "attention_pad_causal": bench_attention(a, True),
           "transformer_step": bench_transformer(a)}
    print(json.dumps(out), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_mha.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
