"""``SparkAsyncDL`` (Estimator) and ``SparkAsyncDLModel`` (Model).

Public API parity with lifeomic/sparkflow/sparkflow/tensorflow_async.py: the same 21 Params with the same
defaults (:176-182), ``@keyword_only`` constructor/``setParams``, the same getters (including the
historically misspelt ``getAqcuireLock``, :245), ``build_optimizer`` with its quirks (options replace
``tfLearningRate``; unknown names fall back to SGD, :32-42), ``_fit`` -> ``HogwildSparkModel.train`` ->
weights JSON -> ``SparkAsyncDLModel`` and ``_transform`` = per-partition ``predict_func``.

Params are declared from a table instead of one statement each; the engine underneath is the H100
parameter-server runtime instead of Flask + TF sessions.
"""
from __future__ import annotations

import json
from typing import Any, Dict, Optional

import numpy as np

from .HogwildSparkModel import HogwildSparkModel
from .ml_util import convert_weights_to_json, predict_func
from .ops.optimizers import OptimizerSpec
from .pipeline_util import PysparkReaderWriter
# genuine pyspark classes when PySpark is importable, the dependency-free stand-ins otherwise (spark/backend.py)
from .spark.backend import (Estimator, HasInputCol, HasLabelCol, HasPredictionCol, Identifiable, MLReadable, MLWritable, Model, Param, Params,
                            SparkContext, TypeConverters, keyword_only)

AVAILABLE_OPTIMIZERS = ("adam", "rmsprop", "momentum", "adadelta", "adagrad", "gradient_descent", "adagrad_da", "ftrl",
                        "proximal_adagrad", "proximal_gradient_descent")


def build_optimizer(optimizer_name: str, learning_rate: float, optimizer_options: Optional[Dict[str, Any]]) -> OptimizerSpec:
    """Name + options -> optimizer.  With ``optimizer_options=None`` the learning rate comes from
    ``learning_rate`` (momentum additionally defaults to 0.9); given options are used verbatim and
    ``learning_rate`` is ignored, exactly like the reference."""
    if optimizer_options is None:
        optimizer_options = {"learning_rate": learning_rate, "use_locking": False}
        if optimizer_name == "momentum":
            optimizer_options["momentum"] = 0.9
    name = optimizer_name if optimizer_name in AVAILABLE_OPTIMIZERS else "gradient_descent"
    return OptimizerSpec.from_tf_kwargs(name, optimizer_options)


def handle_data(data, inp_col: str, label_col: Optional[str]):
    feat = data[inp_col]
    feat = np.asarray(feat.toArray() if hasattr(feat, "toArray") else feat)
    if label_col is None:
        return feat
    return feat, data[label_col]


def _declare(cls, specs):
    """Attach ``Param`` class attributes + ``get<Name>`` accessors from a (name, converter) table."""
    for name, conv in specs:
        setattr(cls, name, Param(Params._dummy(), name, "", typeConverter=conv))
        getter = "get" + name[0].upper() + name[1:]
        if not hasattr(cls, getter):
            setattr(cls, getter, (lambda n: lambda self: self.getOrDefault(getattr(self, n)))(name))
    return cls


_S, _I, _F, _B = TypeConverters.toString, TypeConverters.toInt, TypeConverters.toFloat, TypeConverters.toBoolean

_MODEL_PARAMS = [("modelJson", _S), ("modelWeights", _S), ("tfOutput", _S), ("tfInput", _S), ("tfDropout", _S), ("toKeepDropout", _B)]
_MODEL_DEFAULTS = dict(modelJson=None, inputCol="encoded", predictionCol="predicted", tfOutput=None, tfInput=None,
                       modelWeights=None, tfDropout=None, toKeepDropout=False)

_ESTIMATOR_PARAMS = [("tensorflowGraph", _S), ("tfInput", _S), ("tfOutput", _S), ("tfLabel", _S), ("tfOptimizer", _S),
                     ("tfLearningRate", _F), ("iters", _I), ("partitions", _I), ("miniBatchSize", _I), ("miniStochasticIters", _I),
                     ("verbose", _I), ("acquireLock", _B), ("shufflePerIter", _B), ("tfDropout", _S), ("toKeepDropout", _B),
                     ("partitionShuffles", _I), ("optimizerOptions", _S), ("port", _I)]
_ESTIMATOR_DEFAULTS = dict(inputCol="transformed", tensorflowGraph="", tfInput="x:0", tfLabel=None, tfOutput="out/Sigmoid:0",
                           tfOptimizer="adam", tfLearningRate=.01, partitions=5, miniBatchSize=128, miniStochasticIters=-1,
                           shufflePerIter=True, tfDropout=None, acquireLock=False, verbose=0, iters=1000, toKeepDropout=False,
                           predictionCol="predicted", labelCol=None, partitionShuffles=1, optimizerOptions=None, port=5000)


class SparkAsyncDLModel(Model, HasInputCol, HasPredictionCol, PysparkReaderWriter, MLReadable, MLWritable, Identifiable):
    """Fitted model: graph JSON + weights JSON; ``transform`` adds the prediction column."""

    @keyword_only
    def __init__(self, inputCol=None, modelJson=None, modelWeights=None, tfInput=None, tfOutput=None, tfDropout=None,
                 toKeepDropout=None, predictionCol=None):
        super(SparkAsyncDLModel, self).__init__()
        self._setDefault(**_MODEL_DEFAULTS)
        self.setParams(**self._input_kwargs)

    @keyword_only
    def setParams(self, inputCol=None, modelJson=None, modelWeights=None, tfInput=None, tfOutput=None, tfDropout=None,
                  toKeepDropout=None, predictionCol=None):
        return self._set(**self._input_kwargs)

    def _transform(self, dataset):
        g = self.getOrDefault
        inp, out = g(self.inputCol), g(self.predictionCol)
        mod_json, mod_weights = g(self.modelJson), g(self.modelWeights)
        tf_input, tf_output, tf_dropout, keep = g(self.tfInput), g(self.tfOutput), g(self.tfDropout), g(self.toKeepDropout)
        return dataset.rdd.mapPartitions(
            lambda rows: predict_func(rows, mod_json, out, mod_weights, inp, tf_output, tf_input, tf_dropout, keep)).toDF()


_declare(SparkAsyncDLModel, _MODEL_PARAMS)


class SparkAsyncDL(Estimator, HasInputCol, HasPredictionCol, HasLabelCol, PysparkReaderWriter, MLReadable, MLWritable, Identifiable):
    """Asynchronous deep-learning Estimator.

    inputCol / labelCol / predictionCol: DataFrame columns.  tensorflowGraph: MetaGraphDef JSON from
    ``build_graph``.  tfInput / tfLabel / tfOutput: tensor names.  tfOptimizer + tfLearningRate or
    optimizerOptions (JSON from ``graph_utils.build_*_config``).  iters, partitions, miniBatchSize
    (-1 = whole partition), miniStochasticIters (-1 = sweep the partition), shufflePerIter, acquireLock
    (RW-locked instead of Hogwild), partitionShuffles, verbose, tfDropout / toKeepDropout, port.
    """

    @keyword_only
    def __init__(self, inputCol=None, tensorflowGraph=None, tfInput=None, tfLabel=None, tfOutput=None, tfOptimizer=None,
                 tfLearningRate=None, iters=None, predictionCol=None, partitions=None, miniBatchSize=None,
                 miniStochasticIters=None, acquireLock=None, shufflePerIter=None, tfDropout=None, toKeepDropout=None,
                 verbose=None, labelCol=None, partitionShuffles=None, optimizerOptions=None, port=None):
        super(SparkAsyncDL, self).__init__()
        self._setDefault(**_ESTIMATOR_DEFAULTS)
        self.setParams(**self._input_kwargs)

    @keyword_only
    def setParams(self, inputCol=None, tensorflowGraph=None, tfInput=None, tfLabel=None, tfOutput=None, tfOptimizer=None,
                  tfLearningRate=None, iters=None, predictionCol=None, partitions=None, miniBatchSize=None,
                  miniStochasticIters=None, acquireLock=None, shufflePerIter=None, tfDropout=None, toKeepDropout=None,
                  verbose=None, labelCol=None, partitionShuffles=None, optimizerOptions=None, port=None):
        return self._set(**self._input_kwargs)

    def getAqcuireLock(self):          # sic – public name in the reference
        return self.getOrDefault(self.acquireLock)

    def _fit(self, dataset):
        inp_col, label = self.getInputCol(), self.getLabelCol()
        graph_json = self.getTensorflowGraph()
        opts = self.getOptimizerOptions()
        optimizer = build_optimizer(self.getTfOptimizer(), self.getTfLearningRate(), json.loads(opts) if opts is not None else None)
        partitions = self.getPartitions()

        rdd = dataset.rdd.map(lambda row: handle_data(row, inp_col, label))
        if partitions < rdd.getNumPartitions():
            rdd = rdd.coalesce(partitions)

        sc = SparkContext._active_spark_context or SparkContext.getOrCreate()
        port = self.getPort()
        spark_model = HogwildSparkModel(
            tensorflowGraph=graph_json, iters=self.getIters(), tfInput=self.getTfInput(), tfLabel=self.getTfLabel(),
            optimizer=optimizer, master_url=str(sc.getConf().get("spark.driver.host")) + ":" + str(port),
            acquire_lock=self.getAqcuireLock(), mini_batch=self.getMiniBatchSize(),
            mini_stochastic_iters=self.getMiniStochasticIters(), shuffle=self.getShufflePerIter(), verbose=self.getVerbose(),
            partition_shuffles=self.getPartitionShuffles(), port=port)
        weights = spark_model.train(rdd)
        self.last_training_counters = getattr(spark_model, "counters", None)

        return SparkAsyncDLModel(inputCol=inp_col, modelJson=graph_json, modelWeights=convert_weights_to_json(weights),
                                 tfOutput=self.getTfOutput(), tfInput=self.getTfInput(), tfDropout=self.getTfDropout(),
                                 toKeepDropout=self.getToKeepDropout(), predictionCol=self.getPredictionCol())


_declare(SparkAsyncDL, _ESTIMATOR_PARAMS)
