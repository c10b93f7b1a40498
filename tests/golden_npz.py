"""Golden vectors stored as several .npz parts (every file stays under 1 MB), loaded back as one mapping.

golden_<name>.npz holds the recorded outputs; golden_<name>_bert0.npz, _bert1.npz, ... hold the tiny seeded checkpoint they
were recorded with, split by layer.  A long-context run records its outputs only and shares the checkpoint of the short run
it was made from (weights_from)."""
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class Golden(dict):
    @property
    def files(self):
        return list(self.keys())


def _parts(name):
    yield os.path.join(GOLD, f"{name}.npz")
    i = 0
    while os.path.exists(path := os.path.join(GOLD, f"{name}_bert{i}.npz")):
        yield path
        i += 1


def load(name: str, weights_from: str = None) -> Golden:
    """every part of golden_<name>; with weights_from, the checkpoint tensors (bert_*, not bert_config) of that run too"""
    g = Golden()
    for path in _parts(name):
        with np.load(path) as z:
            g.update({k: z[k] for k in z.files})
    if weights_from is not None:
        w = load(weights_from)
        g.update({k: w[k] for k in w.files if k.startswith("bert_") and k != "bert_config"})
    return g
