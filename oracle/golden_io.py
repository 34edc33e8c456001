"""Golden vectors larger than 1 MB are stored as several .npz files: <name>.npz plus <name>.<part>.npz.
load() returns the union of their arrays as one dict."""
from pathlib import Path

import numpy as np


def load(path) -> dict:
    path = Path(path)
    out = dict(np.load(path))
    for part in sorted(path.parent.glob(path.stem + ".*.npz")):
        out.update(np.load(part))
    return out
