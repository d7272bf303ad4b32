"""The Cora citation graph at the reference's import path ``deep_recommenders.datasets.cora``.

Mirrors reference datasets/cora.py: ``Cora(extract_path)`` reads ``<extract_path>/cora/cora.content`` (paper id, 1433
binary word features, class name per line) and ``cora.cites`` (cited id, citing id per line).  The methods return what
the reference's return, bit for bit under the same ``np.random.seed``: the row-normalised sparse features, the
symmetrised citation graph (a citation present in both directions keeps the value 2 that the reference's
``graph + graph.T - diag`` gives it), the D^-1/2 (A + I) D^-1/2 graph, the per-class training sample (the same
``np.random.choice`` draws), one-hot labels and the train / validation / test split (the validation nodes in the
iteration order of the reference's ``set`` difference).  ``np.str`` / ``np.bool``, which current numpy no longer has,
are ``str`` / ``bool``.  There is no network here: missing files raise ``RuntimeError`` (the reference downloads
them); ``write_synthetic_cora`` writes a seeded graph in Cora's format instead.

scipy is imported by this module only (the reference's own dependency); the rest of the package does not need it.
"""
from __future__ import annotations

import os

import numpy as np
import scipy.sparse as sp

CORA_CLASSES = ["Case_Based", "Genetic_Algorithms", "Neural_Networks", "Probabilistic_Methods",
                "Reinforcement_Learning", "Rule_Learning", "Theory"]


class Cora:

    def __init__(self, extract_path="."):
        self._extract_path = extract_path
        self._cora_path = os.path.join(extract_path, "cora")
        self._cora_cites = os.path.join(self._cora_path, "cora.cites")
        self._cora_content = os.path.join(self._cora_path, "cora.content")
        if not (os.path.exists(self._cora_cites) and os.path.exists(self._cora_content)):
            raise RuntimeError(f"no network in this environment: place cora/cora.content and cora/cora.cites under "
                               f"{os.path.abspath(extract_path)} (or write a synthetic graph with write_synthetic_cora)")
        self._cora_classes = list(CORA_CLASSES)

    @property
    def num_classes(self):
        return len(self._cora_classes)

    def load_content(self, normalize=True):
        """(paper ids [N] str, features [N, words] float32 sparse, row-normalised by default, labels [N] str)."""
        table = np.genfromtxt(self._cora_content, dtype=str)
        ids, labels = table[:, 0], table[:, -1]
        features = sp.csr_matrix(table[:, 1:-1], dtype=np.float32)
        if normalize is True:
            features /= features.sum(axis=1).reshape(-1, 1)
        return ids, features, labels

    def build_graph(self, nodes):
        """Symmetric float32 adjacency [N, N] of the citations between `nodes` (paper ids in row order)."""
        position = {int(paper): row for row, paper in enumerate(nodes)}
        cites = np.genfromtxt(self._cora_cites, dtype=np.int32)
        pairs = np.array([position.get(paper) for paper in cites.flatten()], dtype=np.int32).reshape(cites.shape)
        n = nodes.shape[0]
        graph = sp.coo_matrix((np.ones(pairs.shape[0]), (pairs[:, 0], pairs[:, 1])), shape=(n, n), dtype=np.float32)
        graph += graph.T - sp.diags(graph.diagonal())
        return graph

    @staticmethod
    def spectral_graph(graph):
        """D^-1/2 (A + I) D^-1/2 as CSR, D the row sums of A + I."""
        looped = graph + sp.eye(graph.shape[0])
        d = sp.diags(np.power(np.array(looped.sum(1)), -0.5).flatten(), 0)
        return looped.dot(d).transpose().dot(d).tocsr()

    def sample_train_nodes(self, labels, num_per_class=20):
        """`num_per_class` distinct nodes of every class, classes in order (np.random.choice without replacement)."""
        picked = []
        for name in self._cora_classes:
            members = np.where(labels == name)[0]
            picked += np.random.choice(members, num_per_class, replace=False).tolist()
        return picked

    def encode_labels(self, labels):
        """One-hot int32 [N, num_classes] in the class order above."""
        eye = np.eye(len(self._cora_classes))
        rows = {name: eye[i] for i, name in enumerate(self._cora_classes)}
        return np.array([rows.get(label) for label in labels], dtype=np.int32)

    def split_labels(self, labels, num_valid_nodes=500):
        """((train_labels, train_mask), (valid_labels, valid_mask), (test_labels, test_mask)): labels [N, classes]
        int32, zero outside the split, masks [N] bool.  Train is a fresh sample_train_nodes draw; validation is the
        first `num_valid_nodes` of the other nodes in set-difference order, test the rest."""
        n = labels.shape[0]
        train = self.sample_train_nodes(labels)
        rest = list(set(np.arange(n)) - set(train))
        valid, test = rest[:num_valid_nodes], rest[num_valid_nodes:]
        onehot = self.encode_labels(labels)

        def part(index):
            mask = np.zeros(n)
            mask[index] = 1
            out = np.zeros(onehot.shape, dtype=np.int32)
            out[index] = onehot[index]
            return out, np.array(mask, dtype=bool)

        return part(train), part(valid), part(test)


def write_synthetic_cora(path, seed, num_papers=2708, num_words=1433, num_cites=5429, words_per_paper=18,
                         within_class=0.85, topical_words=0.7):
    """Write ``<path>/cora/cora.content`` and ``cora.cites`` in Cora's text format, seeded, with planted classes.

    Defaults are Cora's shape (2708 papers, 1433 binary word features, 5429 citations, 7 classes).  Each paper gets a
    class uniformly at random; a fraction ``within_class`` of the citations join two papers of one class, and a
    fraction ``topical_words`` of each paper's words come from a block of the vocabulary owned by its class.  Every
    paper has at least one word; there are no self-citations and no repeated (cited, citing) pair.  A GCN learns the
    classes from this well above chance.  Returns ``path``."""
    rng = np.random.default_rng(seed)
    k = len(CORA_CLASSES)
    ids = rng.choice(np.arange(1, 50 * num_papers), size=num_papers, replace=False)
    cls = rng.integers(0, k, size=num_papers)
    block = num_words // k
    words = np.zeros((num_papers, num_words), dtype=np.int8)
    for p in range(num_papers):
        n_topical = rng.binomial(words_per_paper, topical_words)
        own = cls[p] * block + rng.integers(0, block, size=n_topical)
        other = rng.integers(0, num_words, size=words_per_paper - n_topical)
        words[p, np.concatenate([own, other])] = 1
    members = [np.flatnonzero(cls == c) for c in range(k)]
    edges = set()
    while len(edges) < num_cites:
        a = int(rng.integers(0, num_papers))
        if rng.random() < within_class:
            b = int(rng.choice(members[cls[a]]))
        else:
            b = int(rng.integers(0, num_papers))
        if a != b:
            edges.add((a, b))
    root = os.path.join(path, "cora")
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "cora.content"), "w") as f:
        for p in range(num_papers):
            f.write("\t".join([str(ids[p]), *map(str, words[p]), CORA_CLASSES[cls[p]]]) + "\n")
    with open(os.path.join(root, "cora.cites"), "w") as f:
        for a, b in sorted(edges):
            f.write(f"{ids[a]}\t{ids[b]}\n")
    return path
