"""Load a pre-trained TensorFlow checkpoint (``<path>.meta`` + V2 bundle) as a ``SparkAsyncDLModel``.

API parity with lifeomic/sparkflow/sparkflow/tensorflow_model_loader.py:8-45, implemented without
TensorFlow: the binary MetaGraphDef is decoded by ``graph.pbwire`` and the ``.index`` / ``.data``
bundle by the native TF-bundle reader (``io.bundle``).
"""
from __future__ import annotations

import json
import os

from .graph import pbwire
from .graph.ir import GraphIR
from .io.bundle import read_bundle, read_checkpoint_state, write_bundle, write_checkpoint_state
from .spark.ml.base import PipelineModel
from .tensorflow_async import SparkAsyncDLModel


def load_tensorflow_model(path, inputCol, tfInput, tfOutput, predictionCol="predicted", tfDropout=None, toKeepDropout=False):
    with open(path + ".meta", "rb") as fh:
        meta = pbwire.decode("MetaGraphDef", fh.read())
    ckpt_dir = os.path.dirname(path) or "."
    prefix = read_checkpoint_state(ckpt_dir) or path      # ``tf.train.latest_checkpoint`` of the directory
    tensors = read_bundle(prefix)
    ir = GraphIR.from_metagraph(meta)
    weights = []
    for v in ir.trainable:
        if v.name not in tensors:
            raise KeyError(f"variable '{v.name}' is missing from checkpoint {prefix}")
        weights.append(tensors[v.name].reshape(v.shape).tolist())
    return SparkAsyncDLModel(inputCol=inputCol, modelJson=json.dumps(meta), modelWeights=json.dumps(weights), tfInput=tfInput,
                             tfOutput=tfOutput, predictionCol=predictionCol, tfDropout=tfDropout, toKeepDropout=toKeepDropout)


def attach_tensorflow_model_to_pipeline(path, pipelineModel, inputCol, tfInput, tfOutput, predictionCol="predicted",
                                        tfDropout=None, toKeepDropout=False):
    spark_model = load_tensorflow_model(path, inputCol, tfInput, tfOutput, predictionCol, tfDropout, toKeepDropout)
    return PipelineModel(stages=[pipelineModel, spark_model])


def save_tensorflow_model(model, path) -> str:
    """The inverse of :func:`load_tensorflow_model` (an extension - the reference can only import): write a fitted
    ``SparkAsyncDLModel`` as a TensorFlow V2 checkpoint that TF-1.x ``Saver.restore`` / ``import_meta_graph`` reads -
    ``<path>.meta`` (binary MetaGraphDef), ``<path>.index`` + ``<path>.data-00000-of-00001`` (one fp32 tensor per
    trainable variable, under its variable name) and the ``checkpoint`` state file next to them.  Returns ``path``."""
    import numpy as np

    graph = model.getOrDefault(model.modelJson)
    meta = json.loads(graph) if isinstance(graph, str) else graph
    weights = json.loads(model.getOrDefault(model.modelWeights))
    ir = GraphIR.from_metagraph(meta)
    if len(weights) != len(ir.trainable):
        raise ValueError(f"the model carries {len(weights)} weight arrays for {len(ir.trainable)} trainable variables")
    tensors = {v.name: np.asarray(w, dtype=np.float32).reshape(v.shape) for v, w in zip(ir.trainable, weights)}
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    write_bundle(path, tensors)
    with open(path + ".meta", "wb") as fh:
        fh.write(pbwire.encode("MetaGraphDef", meta))
    write_checkpoint_state(os.path.dirname(os.path.abspath(path)), os.path.basename(path))
    return path
