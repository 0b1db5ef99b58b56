"""Tensor / batching / prediction utilities (API parity with lifeomic/sparkflow/sparkflow/ml_util.py).

Differences by design: weights are bound by name to the parsed graph (no per-call assign ops – the
reference leaks a placeholder+assign pair per variable per pull, ml_util.py:16-28), and prediction
runs the compiled sm_90a forward plan when a GPU is present.
"""
from __future__ import annotations

import json
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .graph.executor import GraphProgram
from .graph.ir import GraphIR

_SESSION_WEIGHTS: Dict[int, List[np.ndarray]] = {}


def _rows_to_array(values: Sequence[Any]) -> np.ndarray:
    return np.asarray([np.asarray(v.toArray() if hasattr(v, "toArray") else v, dtype=np.float32).reshape(-1) for v in values],
                      dtype=np.float32)


def tensorflow_get_weights(vs=None, session=None):
    """Values of the trainable variables of the default tfcompat session."""
    from .graph.tfcompat import get_default_session, trainable_variables

    sess = session or get_default_session()
    vs = vs or trainable_variables()
    return [sess._values[v._name].detach().cpu().numpy() for v in vs]


def tensorflow_set_weights(weights, vs=None, session=None):
    from .graph.tfcompat import get_default_session, trainable_variables

    sess = session or get_default_session()
    vs = vs or trainable_variables()
    for var, value in zip(vs, weights):
        sess.set_variable(var._name, np.asarray(value))


def convert_weights_to_json(weights: Sequence[np.ndarray]) -> str:
    return json.dumps([np.asarray(w).tolist() for w in weights])


def convert_json_to_weights(json_weights: str) -> List[np.ndarray]:
    return [np.asarray(x) for x in json.loads(json_weights)]


def calculate_weights(collected_weights: Sequence[Sequence[np.ndarray]]) -> List[np.ndarray]:
    """Element-wise mean of several weight lists (kept for API parity; unused by the async trainer)."""
    n = len(collected_weights)
    return [sum(np.asarray(ws[i]) for ws in collected_weights) / n for i in range(len(collected_weights[0]))]


def handle_features(data: Iterable, is_supervised: bool = False) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    features, labels = [], []
    for item in data:
        if is_supervised:
            x, y = item
            if isinstance(y, (int, float, np.integer, np.floating)):
                y = [y]
            labels.append(np.asarray(y.toArray() if hasattr(y, "toArray") else y, dtype=np.float32).reshape(-1))
        else:
            x = item
        features.append(np.asarray(x.toArray() if hasattr(x, "toArray") else x, dtype=np.float32).reshape(-1))
    feats = np.asarray(features, dtype=np.float32)
    return feats, (np.asarray(labels, dtype=np.float32) if is_supervised else None)


def handle_feed_dict(train, tfInput, tfLabel=None, labels=None, mini_batch_size=-1, idx=None):
    n = train.shape[0]
    if mini_batch_size > n:
        mini_batch_size = n - 1
    if mini_batch_size <= 0:
        sel: Any = slice(0, n)
    elif idx is not None:
        sel = slice(idx, idx + mini_batch_size)
    else:
        sel = np.random.choice(n, mini_batch_size, replace=False)
    feed = {tfInput: train[sel]}
    if tfLabel is not None:
        feed[tfLabel] = labels[sel]
    return feed


def handle_shuffle(features, labels):
    perm = np.random.permutation(features.shape[0])
    return features[perm], (labels[perm] if labels is not None else None)


# ---------------------------------------------------------------------------------------------
_PREDICTORS: Dict[Tuple[int, str, str], Any] = {}


def run_inference(graph_json: str, weights: Sequence[np.ndarray], features: np.ndarray, tf_input: str, tf_output: str,
                  tf_dropout: Optional[str] = None, to_keep_dropout: bool = False) -> np.ndarray:
    """Forward pass of ``tf_output`` for a feature matrix.  GPU: compiled forward plan (wgmma GEMMs with
    fused bias/activation, ArgMax kernel); otherwise (or for graphs outside the compiled family) the
    interpreter."""
    import torch

    ir = GraphIR.from_metagraph(graph_json)
    feats = np.ascontiguousarray(features, dtype=np.float32)
    if torch.cuda.is_available() and tf_dropout is None:
        from .models.compiler import UnsupportedGraph, compile_graph

        try:
            from .parallel.plan_builder import check_grammar

            lp = compile_graph(ir, tf_input, None, tf_output, need_loss=False)
            check_grammar(lp)
            if lp.output is not None and lp.output.layer >= 0 and lp.layers[lp.output.layer].kind == "dense":
                from .ops.layout import ParamLayout
                from .ops.optimizers import OptimizerSpec
                from .parallel.device_engine import DeviceWorker, MasterState

                dense_idx = [i for i, l in enumerate(lp.layers) if l.kind == "dense"]
                upto = dense_idx.index(lp.output.layer)
                spec = OptimizerSpec("gradient_descent", {"lr": 0.0})
                lay = ParamLayout.build(ir.param_shapes())
                dev = torch.device("cuda", torch.cuda.current_device())
                master = MasterState(lay, spec, dev)
                try:
                    master.load_weights(list(weights))
                    worker = DeviceWorker.for_inference(ir, lp, spec, master)
                    return worker.predict(feats, upto=upto, post=lp.output.post)
                finally:
                    master.close()
        except UnsupportedGraph:
            pass
    prog = GraphProgram(ir, "cuda" if torch.cuda.is_available() else "cpu")
    feed: Dict[str, Any] = {tf_input: feats}
    if tf_dropout is not None:
        feed[tf_dropout] = np.asarray(1.0 if to_keep_dropout else 0.0, dtype=np.float32)
    return prog.forward(tf_output, feed, list(weights)).detach().cpu().numpy()


def predict_func(rows, graph_json, prediction, graph_weights, inp, activation, tf_input, tf_dropout=None, to_keep_dropout=False):
    """Per-partition prediction: adds ``prediction`` to every row (float for scalar outputs, a
    ``DenseVector`` otherwise) – reference: ml_util.py:54-83."""
    from .spark.backend import Row, Vectors          # genuine pyspark classes when PySpark is installed

    rows = [r.asDict() for r in rows]
    if not rows:
        return []
    weights = [np.asarray(x, dtype=np.float32) for x in json.loads(graph_weights)]
    feats = _rows_to_array([r[inp] for r in rows])
    pred = run_inference(graph_json, weights, feats, tf_input, activation, tf_dropout, to_keep_dropout)
    out = []
    for r, p in zip(rows, pred):
        p = np.asarray(p)
        r[prediction] = float(p.reshape(-1)[0]) if p.size == 1 else Vectors.dense(p.astype(np.float64))
        out.append(Row(**r))
    return out
