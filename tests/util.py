"""Shared helpers for the tests (not product code)."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_v1.npz"))


def ref_data(name):
    """Bytes of a data file shipped with the reference release (query.hhm, cs219.lib), stored under tests/golden."""
    with np.load(os.path.join(ROOT, "tests", "golden", "refdata_v1.npz")) as z:
        return z[name.replace(".", "_")].tobytes()


def ref_data_file(name, directory):
    """ref_data(name) written to directory/name; returns the path as a string."""
    path = os.path.join(str(directory), name)
    with open(path, "wb") as f:
        f.write(ref_data(name))
    return path


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def rasterize_exclusion(Lq, Lt, i_steps, j_steps, nsteps):
    """Numpy restatement of Viterbi::ExcludeAlignment (src/hhviterbi.cpp:61-77) for test inputs."""
    m = np.zeros((Lq + 1, Lt + 1), np.uint8)
    for s in range(1, nsteps):
        i, j = int(i_steps[s]), int(j_steps[s])
        m[max(i - 40, 1):min(i + 40, Lq) + 1, j] = 1
        m[i, max(j - 40, 1):min(j + 40, Lt) + 1] = 1
    return m
