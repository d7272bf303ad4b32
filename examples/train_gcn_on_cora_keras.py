"""The reference's examples/train_gcn_on_cora_keras.py.

Same calls in the same order: Cora() -> load_content -> build_graph -> spectral_graph -> sample_train_nodes (whose draw
is discarded but consumes the RNG, as in the reference) -> split_labels; GCN(32) then GCN(7, activation="softmax");
Adam(0.01), categorical cross-entropy, weighted_metrics=["acc"]; full-batch fit with the train mask as sample weight,
validation on the validation mask, EarlyStopping(patience=3); the test loss and accuracy printed at the end.  There is
no functional `Input`, so the model is a small `Model` subclass, and the spectral graph is prepared on the device once.
The Cora files are read from ./cora when they exist; otherwise a seeded synthetic graph of Cora's shape is written to a
temporary directory and read through the same loader.

    python examples/train_gcn_on_cora_keras.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deep_recommenders.datasets import Cora, write_synthetic_cora  # noqa: E402
from deep_recommenders.keras.layers import Model  # noqa: E402
from deep_recommenders.keras.models.retrieval import GCN  # noqa: E402
from deep_recommenders_b200 import ops  # noqa: E402
from deep_recommenders_b200.keras.engine import Adam, EarlyStopping  # noqa: E402


class GCNClassifier(Model):
    def __init__(self, num_classes):
        super().__init__()
        self.gcn1 = GCN(32)
        self.gcn2 = GCN(num_classes, activation="softmax")
        self.built = True

    def call(self, inputs, **kwargs):
        g, feats = inputs
        return self.gcn2(self.gcn1(feats, g), g)


def train_model(extract_path=".", epochs=200, seed=0, verbose=2):
    np.random.seed(seed)
    torch.manual_seed(seed)
    cora = Cora(extract_path)
    ids, features, labels = cora.load_content()
    graph = cora.build_graph(ids)
    spectral_graph = cora.spectral_graph(graph)
    cora.sample_train_nodes(labels)
    train, valid, test = cora.split_labels(labels)

    g = ops.CSRAdjacency.from_any(spectral_graph)
    feats = torch.from_numpy(np.asarray(features.todense(), dtype=np.float32)).cuda()
    model = GCNClassifier(cora.num_classes)
    model.compile(optimizer=Adam(0.01), loss="categorical_crossentropy", weighted_metrics=["acc"])

    train_labels, train_mask = train
    valid_labels, valid_mask = valid
    test_labels, test_mask = test
    batch_size = graph.shape[0]

    history = model.fit([g, feats], train_labels, sample_weight=train_mask,
                        validation_data=([g, feats], valid_labels, valid_mask), batch_size=batch_size, epochs=epochs,
                        shuffle=False, verbose=verbose, callbacks=[EarlyStopping(patience=3)])
    eval_results = model.evaluate([g, feats], test_labels, sample_weight=test_mask, batch_size=batch_size, verbose=0)
    print("Test Loss: {:.4f}".format(eval_results["loss"]))
    print("Test Accuracy: {:.4f}".format(eval_results["acc"]))
    return history, eval_results


if __name__ == "__main__":
    if os.path.exists(os.path.join("cora", "cora.content")):
        train_model(".")
    else:
        with tempfile.TemporaryDirectory() as tmp:
            print(f"./cora not found: training on a synthetic graph of Cora's shape (seed 0)")
            train_model(write_synthetic_cora(tmp, seed=0))
