"""Snapshot / resume of the parameter server state in TensorFlow's V2 bundle layout.

The reference never checkpoints during training: the master lives only in the Flask process' memory
(SURVEY.md section 5).  Here the master's parameters AND optimizer slots can be written as a TF checkpoint with
the names TF itself would use (``<var>``, ``<var>/Adam``, ``<var>/Adam_1``, ``beta1_power``, ``beta2_power`` –
compare the keys of lifeomic/sparkflow/tests/test_model/to_load.index), so a snapshot is loadable by
``load_tensorflow_model`` (and by TensorFlow), and training can resume from it with identical optimizer state.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from ..io.bundle import read_bundle, write_bundle, write_checkpoint_state
from ..ops.optimizers import OptimizerSpec

STEP_KEY = "sparkflow_b200/optimizer_step"


def save_master_state(prefix: str, var_names: Sequence[str], weights: Sequence[np.ndarray], slots: Sequence[Sequence[np.ndarray]],
                      spec: OptimizerSpec, step: int, graph_json: Optional[str] = None) -> str:
    tensors: Dict[str, np.ndarray] = {}
    for name, w in zip(var_names, weights):
        tensors[name] = np.asarray(w, dtype=np.float32)
    for si, slot_name in enumerate(spec.slot_names()[: len(slots)]):
        for name, arr in zip(var_names, slots[si]):
            tensors[f"{name}/{slot_name}"] = np.asarray(arr, dtype=np.float32)
    if spec.name == "adam":
        b1, b2 = float(spec.hyper.get("beta1", 0.9)), float(spec.hyper.get("beta2", 0.999))
        tensors["beta1_power"] = np.asarray(b1 ** (step + 1), dtype=np.float32)
        tensors["beta2_power"] = np.asarray(b2 ** (step + 1), dtype=np.float32)
    tensors[STEP_KEY] = np.asarray(step, dtype=np.int64)
    write_bundle(prefix, tensors)
    write_checkpoint_state(os.path.dirname(os.path.abspath(prefix)), os.path.basename(prefix))
    if graph_json is not None:
        from ..graph.tfcompat import MetaGraphDef
        import json

        with open(prefix + ".meta", "wb") as fh:
            fh.write(MetaGraphDef(json.loads(graph_json)).SerializeToString())
    return prefix


def load_master_state(prefix: str, var_names: Sequence[str], spec: OptimizerSpec) -> Tuple[List[np.ndarray], List[List[np.ndarray]], int]:
    tensors = read_bundle(prefix)
    weights = []
    for name in var_names:
        if name not in tensors:
            raise KeyError(f"checkpoint {prefix} has no variable '{name}'")
        weights.append(tensors[name])
    slots: List[List[np.ndarray]] = []
    for si, slot_name in enumerate(spec.slot_names()):
        keys = [f"{n}/{slot_name}" for n in var_names]
        if all(k in tensors for k in keys):
            slots.append([tensors[k] for k in keys])
        else:
            break
    step = int(tensors[STEP_KEY]) if STEP_KEY in tensors else 0
    return weights, slots, step
