"""``tf.train``: optimizer descriptors, MetaGraph import/export and a TF-bundle ``Saver``.

The reference hands ``tf.train.*Optimizer`` instances to the parameter server, which only ever calls
``optimizer.apply_gradients`` on the master (lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:194).
Here the optimizer classes are thin constructors of :class:`OptimizerSpec`, which is what the master
(torch on CPU, the fused push kernel on H100) consumes.
"""
from __future__ import annotations

import os
from typing import Any, Dict, List, Optional

import numpy as np

from ...ops.optimizers import OptimizerSpec
from . import core
from .core import MetaGraphDef, export_meta_graph  # noqa: F401  (re-export)


class Optimizer(OptimizerSpec):
    _tf_name = "gradient_descent"

    def __init__(self, **kwargs):
        spec = OptimizerSpec.from_tf_kwargs(self._tf_name, kwargs)
        super().__init__(name=spec.name, hyper=spec.hyper)

    def minimize(self, loss, global_step=None, var_list=None, name=None):
        g = loss.graph
        op = g.add_node("NoOp", name or type(self).__name__.replace("Optimizer", ""))
        g.add_to_collection(core.GraphKeys.TRAIN_OP, op)
        g.add_to_collection("sparkflow_optimizer", self)
        return op

    def __reduce__(self):
        return (_rebuild, (self.name, dict(self.hyper)))


def _rebuild(name, hyper):
    return OptimizerSpec(name=name, hyper=hyper)


def _mk(cls_name: str, tf_name: str, positional: List[str], defaults: Dict[str, Any]):
    def __init__(self, *args, **kwargs):
        if len(args) > len(positional):
            raise TypeError(f"{cls_name}() takes at most {len(positional)} positional arguments")
        kw = dict(defaults)
        kw.update(dict(zip(positional, args)))
        kw.update(kwargs)
        Optimizer.__init__(self, **kw)

    return type(cls_name, (Optimizer,), {"__init__": __init__, "_tf_name": tf_name})


GradientDescentOptimizer = _mk("GradientDescentOptimizer", "gradient_descent", ["learning_rate", "use_locking", "name"], {})
AdamOptimizer = _mk("AdamOptimizer", "adam", ["learning_rate", "beta1", "beta2", "epsilon", "use_locking", "name"], {"learning_rate": 0.001})
RMSPropOptimizer = _mk("RMSPropOptimizer", "rmsprop", ["learning_rate", "decay", "momentum", "epsilon", "use_locking", "centered", "name"], {})
MomentumOptimizer = _mk("MomentumOptimizer", "momentum", ["learning_rate", "momentum", "use_locking", "name", "use_nesterov"], {})
AdadeltaOptimizer = _mk("AdadeltaOptimizer", "adadelta", ["learning_rate", "rho", "epsilon", "use_locking", "name"], {"learning_rate": 0.001})
AdagradOptimizer = _mk("AdagradOptimizer", "adagrad", ["learning_rate", "initial_accumulator_value", "use_locking", "name"], {})
AdagradDAOptimizer = _mk("AdagradDAOptimizer", "adagrad_da", ["learning_rate", "global_step", "initial_gradient_squared_accumulator_value",
                                                               "l1_regularization_strength", "l2_regularization_strength", "use_locking", "name"], {})
FtrlOptimizer = _mk("FtrlOptimizer", "ftrl", ["learning_rate", "learning_rate_power", "initial_accumulator_value", "l1_regularization_strength",
                                               "l2_regularization_strength", "use_locking", "name"], {})
ProximalAdagradOptimizer = _mk("ProximalAdagradOptimizer", "proximal_adagrad", ["learning_rate", "initial_accumulator_value",
                                                                                 "l1_regularization_strength", "l2_regularization_strength", "use_locking", "name"], {})
ProximalGradientDescentOptimizer = _mk("ProximalGradientDescentOptimizer", "proximal_gradient_descent",
                                       ["learning_rate", "l1_regularization_strength", "l2_regularization_strength", "use_locking", "name"], {})


# ---------------------------------------------------------------------------
# checkpoints
# ---------------------------------------------------------------------------
def latest_checkpoint(checkpoint_dir: str, latest_filename: Optional[str] = None) -> Optional[str]:
    from ...io.bundle import read_checkpoint_state

    return read_checkpoint_state(checkpoint_dir, latest_filename or "checkpoint")


class Saver:
    """Writes / restores TF-V2 bundles (``<prefix>.index`` + ``<prefix>.data-00000-of-00001``) and ``.meta``."""

    def __init__(self, var_list=None, max_to_keep: int = 5, graph: Optional[core.Graph] = None, **_unused):
        self.graph = graph or core.get_default_graph()
        self.var_list = var_list
        if self.graph.saver_def is None:
            self.graph.saver_def = {"filenameTensorName": "save/Const:0", "saveTensorName": "save/control_dependency:0",
                                    "restoreOpName": "save/restore_all", "maxToKeep": max_to_keep, "version": "V2"}

    def _vars(self) -> List[core.Variable]:
        return list(self.var_list) if self.var_list is not None else list(self.graph.variables)

    def save(self, sess, save_path: str, global_step=None, write_meta_graph: bool = True, **_unused) -> str:
        from ...io.bundle import write_bundle, write_checkpoint_state

        prefix = save_path if global_step is None else f"{save_path}-{int(global_step)}"
        tensors = {}
        for v in self._vars():
            if v._name not in sess._values:
                raise ValueError(f"Attempting to use uninitialized value {v._name}")
            tensors[v._name] = sess._values[v._name].detach().cpu().numpy()
        os.makedirs(os.path.dirname(os.path.abspath(prefix)), exist_ok=True)
        write_bundle(prefix, tensors)
        write_checkpoint_state(os.path.dirname(os.path.abspath(prefix)), os.path.basename(prefix))
        if write_meta_graph:
            export_meta_graph(prefix + ".meta", graph=self.graph)
        return prefix

    def restore(self, sess, save_path: str) -> None:
        from ...io.bundle import read_bundle

        if save_path is None:
            raise ValueError("Can't load save_path when it is None.")
        tensors = read_bundle(save_path)
        for v in self._vars():
            if v._name in tensors:
                sess.set_variable(v._name, tensors[v._name])


def import_meta_graph(meta_graph_or_file, clear_devices: bool = False, import_scope=None, **_unused) -> Saver:
    """Rebuilds the default graph from a MetaGraphDef (file path, bytes, JSON text or object)."""
    from ..ir import GraphIR

    if isinstance(meta_graph_or_file, str) and os.path.exists(meta_graph_or_file):
        with open(meta_graph_or_file, "rb") as fh:
            raw = fh.read()
        mg = MetaGraphDef.FromString(raw)
    elif isinstance(meta_graph_or_file, bytes):
        mg = MetaGraphDef.FromString(meta_graph_or_file)
    elif isinstance(meta_graph_or_file, MetaGraphDef):
        mg = meta_graph_or_file
    else:
        import json

        mg = MetaGraphDef(json.loads(meta_graph_or_file) if isinstance(meta_graph_or_file, str) else dict(meta_graph_or_file))
    g = core.get_default_graph()
    ir = GraphIR.from_metagraph(mg.data)
    _load_ir_into_graph(g, ir, mg.data)
    return Saver(graph=g)


def _load_ir_into_graph(g: core.Graph, ir, data: Dict[str, Any]) -> None:
    from .core import Operation, Tensor, Variable, as_dtype

    for nd in data.get("graphDef", {}).get("node", []):
        name = nd["name"]
        if name in g._ops:
            raise ValueError(f"node {name} already exists in the target graph")
        node = dict(nd)
        g.nodes.append(node)
        g._node_index[name] = node
        g._names_in_use[name.lower()] = 1
        irn = ir.nodes[name]
        n_out = 2 if irn.op == "SoftmaxCrossEntropyWithLogits" else 1
        dt_name = irn.attrs.get("dtype") or irn.attrs.get("T") or irn.attrs.get("DstT") or "DT_FLOAT"
        try:
            dt = as_dtype(dt_name.replace("_REF", "") if isinstance(dt_name, str) else "DT_FLOAT")
        except TypeError:
            dt = core.float32
        shapes = irn.attrs.get("_output_shapes") or []
        outs = []
        for i in range(n_out):
            shp = shapes[i] if i < len(shapes) else irn.attrs.get("shape") if irn.op in ("Placeholder", "VariableV2") else None
            t = Tensor(g, name, i, dt, None if shp is None else tuple(shp))
            outs.append(t)
            g._tensors[t.name] = t
        op = Operation(g, node, outs)
        for t in outs:
            t.op = op
        g._ops[name] = op
    trainable = {v.name for v in ir.trainable}
    for v in ir.variables or ir.trainable:
        if v.name not in g._ops:
            continue
        handle = g._tensors[f"{v.name}:0"]
        read = g._tensors.get(f"{v.name}/read:0", handle)
        init_val = g._tensors.get(v.initial_value) if v.initial_value else None
        init_op = g._ops.get(f"{v.name}/Assign")
        var = Variable(g, v.name, core.float32, tuple(v.shape), handle, read, init_val, init_op, v.name in trainable)
        g.variables.append(var)
        g.add_to_collection(core.GraphKeys.GLOBAL_VARIABLES, var)
        if v.name in trainable:
            g.add_to_collection(core.GraphKeys.TRAINABLE_VARIABLES, var)
    for ref in ir.losses:
        if ref in g._tensors:
            g.add_to_collection(core.GraphKeys.LOSSES, g._tensors[ref])
    if data.get("saverDef"):
        g.saver_def = dict(data["saverDef"])
