"""The reference's examples/train_transformer_on_imdb_keras.py on seeded synthetic token sequences.

Same model (Transformer(vocab, 8, n_heads=2, encoder_stack=2, decoder_stack=2, feed_forward_size=50), mean pooled over
the sequence, Dense(2, softmax)), Adam(beta_1=0.9, beta_2=0.98, epsilon=1e-9), categorical cross-entropy,
EarlyStopping(patience=3) and the Noam schedule.  The IMDB download is not available, so each sequence is a
left-zero-padded run of token ids whose label is learnable: class 1 sequences draw their tokens from the upper half of
the vocabulary far more often than class 0 sequences do.  Both the encoder and the decoder read the same ids, as the
reference feeds the review to both.

    python examples/train_transformer_on_synthetic_keras.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deep_recommenders.keras.layers import Dense, Model  # noqa: E402
from deep_recommenders_b200 import ops  # noqa: E402
from deep_recommenders.keras.models.nlp import Transformer  # noqa: E402
from deep_recommenders.keras.models.nlp.transformer import Noam  # noqa: E402
from deep_recommenders_b200.keras.engine import Adam, EarlyStopping  # noqa: E402


def synthetic_batches(vocab_size, max_len, batch_size, seed):
    """Endless (([ids, ids]), one-hot labels) batches; ids [batch, max_len] int64 with 0 as left padding."""
    rng = np.random.default_rng(seed)
    half = vocab_size // 2
    while True:
        y = rng.integers(0, 2, size=batch_size)
        lengths = rng.integers(max_len // 4, max_len + 1, size=batch_size)
        ids = np.zeros((batch_size, max_len), np.int64)
        for b in range(batch_size):
            upper = rng.random(lengths[b]) < (0.9 if y[b] else 0.1)
            tok = np.where(upper, rng.integers(half, vocab_size, lengths[b]), rng.integers(1, half, lengths[b]))
            ids[b, max_len - lengths[b]:] = tok
        x = torch.from_numpy(ids).cuda()
        yield [x, x], np.eye(2, dtype=np.float32)[y]


class TransformerClassifier(Model):
    def __init__(self, vocab_size, max_len, model_dim=8, n_heads=2, encoder_stack=2, decoder_stack=2, ff_size=50,
                 seed=None):
        super().__init__()
        self.transformer = Transformer(vocab_size, model_dim, n_heads=n_heads, encoder_stack=encoder_stack,
                                       decoder_stack=decoder_stack, feed_forward_size=ff_size, seed=seed)
        self.head = Dense(2, activation=None, seed=seed)
        self.built = True

    def call(self, inputs, **kwargs):
        enc, dec = inputs
        pooled = self.transformer(enc, dec).mean(dim=1)           # GlobalAveragePooling1D
        return ops.SoftmaxRowsFn.apply(self.head(pooled))         # Dense(2, activation='softmax')


def train_model(vocab_size=5000, max_len=128, batch_size=128, epochs=10, steps_per_epoch=50, warmup_steps=100,
                seed=0):
    torch.manual_seed(seed)
    model = TransformerClassifier(vocab_size, max_len, seed=seed)
    model.compile(optimizer=Adam(beta_1=0.9, beta_2=0.98, epsilon=1e-9), loss="categorical_crossentropy")
    es = EarlyStopping(patience=3)
    noam = Noam(model_dim=8, warmup_steps=warmup_steps)
    hist = model.fit(synthetic_batches(vocab_size, max_len, batch_size, seed), epochs=epochs,
                     steps_per_epoch=steps_per_epoch,
                     validation_data=lambda: synthetic_batches(vocab_size, max_len, batch_size, seed + 1),
                     validation_steps=5, callbacks=[es, noam], verbose=1)
    return hist


if __name__ == "__main__":
    h = train_model()
    print("loss by epoch:", " ".join(f"{v:.4f}" for v in h["loss"]))
