"""Which Spark do the API classes build on?

The reference *is* a ``pyspark.ml`` Estimator / Model (lifeomic/sparkflow/sparkflow/tensorflow_async.py:51,102) and persists
through the JVM ``JavaMLWriter`` (lifeomic/sparkflow/sparkflow/pipeline_util.py:85-127).  When a genuine PySpark is importable
``SparkAsyncDL`` / ``SparkAsyncDLModel`` / ``PysparkReaderWriter`` derive from ITS classes - they sit in a real
``Pipeline``, take real DataFrames and save through ``JavaMLWriter``; otherwise (this image: no pyspark, no JVM) they
derive from the dependency-free stand-ins under ``sparkflow_b200.spark`` with the same behaviour and on-disk layout.
``SPARKFLOW_FORCE_SHIM=1`` selects the stand-ins even when PySpark is installed.
"""
from __future__ import annotations

import os
import sys

REAL_PYSPARK = False
if os.environ.get("SPARKFLOW_FORCE_SHIM") != "1":
    _mod = sys.modules.get("pyspark")
    if _mod is None or not getattr(_mod, "__sparkflow_shim__", False):
        try:
            import pyspark as _pyspark  # noqa: F401

            REAL_PYSPARK = not getattr(_pyspark, "__sparkflow_shim__", False) and hasattr(_pyspark, "SparkContext")
        except Exception:  # not installed (or half installed: no JVM bindings)
            REAL_PYSPARK = False

if REAL_PYSPARK:
    try:
        from pyspark import SparkContext, keyword_only
        from pyspark.ml import Estimator, Model, Pipeline, PipelineModel
        from pyspark.ml.feature import StopWordsRemover
        from pyspark.ml.linalg import Vectors
        from pyspark.ml.param import Param, Params, TypeConverters
        from pyspark.ml.param.shared import HasInputCol, HasLabelCol, HasPredictionCol
        from pyspark.ml.util import Identifiable, JavaMLReader, JavaMLWriter, MLReadable, MLReader, MLWritable, MLWriter
        from pyspark.sql import Row
    except Exception:
        REAL_PYSPARK = False

if not REAL_PYSPARK:
    from .context import SparkContext, keyword_only  # noqa: F401
    from .ml.base import Estimator, MLReadable, MLReader, MLWritable, MLWriter, Model, Pipeline, PipelineModel  # noqa: F401
    from .ml.feature import StopWordsRemover  # noqa: F401
    from .ml.linalg import Vectors  # noqa: F401
    from .ml.param import HasInputCol, HasLabelCol, HasPredictionCol, Identifiable, Param, Params, TypeConverters  # noqa: F401
    from .sql import Row  # noqa: F401

    JavaMLReader = JavaMLWriter = None


def collect_partitions(rdd):
    """The rows of every partition of ``rdd`` on the driver: the H100 engine trains on the GPUs of the driver's box, the
    partitions are its workers' shards (reference: ``rdd.foreachPartition(handle_model)``, HogwildSparkModel.py:259)."""
    if hasattr(rdd, "partitions") and callable(rdd.partitions):
        return [list(p) for p in rdd.partitions()]          # stand-in RDD
    return [list(p) for p in rdd.glom().collect()]          # genuine pyspark RDD
