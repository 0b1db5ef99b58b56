"""Locate (or synthesise) the MNIST CSV the reference examples read (label + 784 pixel columns)."""
import os

import numpy as np

CANDIDATES = ["examples/mnist_train.csv", "mnist_train.csv"]


def mnist_csv(rows: int = 4000) -> str:
    for c in CANDIDATES:
        if os.path.exists(c):
            return c
    path = "/tmp/sparkflow_b200_synthetic_mnist.csv"
    if not os.path.exists(path):
        rng = np.random.default_rng(0)
        protos = rng.integers(0, 255, (10, 784))
        lab = rng.integers(0, 10, rows)
        px = np.clip(protos[lab] + rng.normal(0, 40, (rows, 784)), 0, 255).astype(np.int64)
        np.savetxt(path, np.concatenate([lab[:, None], px], axis=1), fmt="%d", delimiter=",")
    return path
