"""Golden vectors stored as several .npz parts (every file stays under 1 MB), loaded back as one mapping.

golden_<name>.npz holds the recorded outputs; golden_<name>_bert0.npz / _bert1.npz hold the tiny seeded checkpoint they
were recorded with (layer 1 in _bert1, everything else in _bert0)."""
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class Golden(dict):
    @property
    def files(self):
        return list(self.keys())


def load(name: str) -> Golden:
    g = Golden()
    for suffix in ("", "_bert0", "_bert1"):
        path = os.path.join(GOLD, f"{name}{suffix}.npz")
        if suffix and not os.path.exists(path):
            continue
        with np.load(path) as z:
            g.update({k: z[k] for k in z.files})
    return g
