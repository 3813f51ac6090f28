"""TEST INFRASTRUCTURE ONLY -- golden fixtures under tests/golden/ are stored as NAME.npz plus, for fixtures whose arrays exceed
1 MB together, NAME.partN.npz files (each compressed file < 1 MB; the split is lossless).  load() merges them back."""
import glob
import os

import numpy as np

MAX_FILE_BYTES = 1 << 20


class Fixture(dict):
    """The merged arrays of a fixture; `.files` lists the names, as for the NpzFile of np.load."""

    @property
    def files(self):
        return list(self.keys())


def load(golden_dir, name):
    fx = Fixture(np.load(os.path.join(golden_dir, name + ".npz")))
    for part in sorted(glob.glob(os.path.join(golden_dir, name + ".part*.npz"))):
        fx.update(np.load(part))
    return fx


def save(golden_dir, name, arrays, max_bytes=MAX_FILE_BYTES):
    """Writes arrays as NAME.npz (+ NAME.partN.npz): greedy packing by raw size with half the limit per file as the budget (random
    fp32 data does not compress), so every compressed file stays below max_bytes."""
    for old in glob.glob(os.path.join(golden_dir, name + ".part*.npz")):
        os.remove(old)
    groups, cur, size = [], {}, 0
    for k in sorted(arrays, key=lambda k: np.asarray(arrays[k]).nbytes):
        nb = np.asarray(arrays[k]).nbytes
        assert nb <= max_bytes, "%s.%s alone is %d bytes" % (name, k, nb)
        if cur and size + nb > max_bytes * 0.9:
            groups.append(cur)
            cur, size = {}, 0
        cur[k] = arrays[k]
        size += nb
    groups.append(cur)
    paths = [os.path.join(golden_dir, name + ".npz")] + [os.path.join(golden_dir, "%s.part%d.npz" % (name, i)) for i in range(1, len(groups))]
    for p, g in zip(paths, groups):
        np.savez_compressed(p, **g)
        assert os.path.getsize(p) <= max_bytes, "%s: %d bytes" % (p, os.path.getsize(p))
    return paths
