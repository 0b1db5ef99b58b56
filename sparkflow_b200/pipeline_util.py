"""Persistence of pure-python pipeline stages through a ``StopWordsRemover`` *carrier*.

Format parity with lifeomic/sparkflow/sparkflow/pipeline_util.py:16-127: a stage is ``dill``-pickled,
zlib-compressed, written as ONE string of decimal byte values each followed by ``','``, and stored as
``stopWords = [payload, GUID]`` of a ``StopWordsRemover`` that carries the python object's uid; loading
recognises carriers by the GUID in the last stop word.  The byte<->decimal codec is native
(``_host.so``) with a pure-python fallback.
"""
from __future__ import annotations

import zlib
from typing import List

import dill

from .spark.backend import REAL_PYSPARK, JavaMLReader, JavaMLWriter, MLReader, MLWriter, Pipeline, PipelineModel, StopWordsRemover


class PysparkObjId(object):
    """Constants identifying carrier stages."""

    @staticmethod
    def _getPyObjId() -> str:
        return "4c1740b00d3c4ff6806a1402321572cb"

    @staticmethod
    def _getCarrierClass(javaName: bool = False):
        return "org.apache.spark.ml.feature.StopWordsRemover" if javaName else StopWordsRemover


def _encode_bytes(raw: bytes) -> str:
    try:
        from .ops.native import host_ext

        return host_ext().bytes_to_decimal_csv(raw)
    except Exception:
        return "".join("%d," % b for b in raw)


def _decode_bytes(text: str) -> bytes:
    try:
        from .ops.native import host_ext

        return bytes(host_ext().decimal_csv_to_bytes(text))
    except Exception:
        return bytes(int(t) for t in text.split(",")[:-1])


def dump_byte_array(py_obj) -> List[str]:
    return [_encode_bytes(zlib.compress(dill.dumps(py_obj)))]


def load_byte_array(stop_words: List[str]):
    return dill.loads(zlib.decompress(_decode_bytes(stop_words[0])))


class PysparkPipelineWrapper(object):
    """Turns carrier stages of a loaded ``Pipeline`` / ``PipelineModel`` back into python objects."""

    @staticmethod
    def unwrap(pipeline):
        if not isinstance(pipeline, (Pipeline, PipelineModel)):
            raise TypeError("Cannot recognize a pipeline of type %s." % type(pipeline))
        stages = pipeline.getStages() if isinstance(pipeline, Pipeline) else pipeline.stages
        for i, stage in enumerate(stages):
            if isinstance(stage, (Pipeline, PipelineModel)):
                stages[i] = PysparkPipelineWrapper.unwrap(stage)
            elif isinstance(stage, PysparkObjId._getCarrierClass()) and stage.getStopWords() \
                    and stage.getStopWords()[-1] == PysparkObjId._getPyObjId():
                stages[i] = load_byte_array(stage.getStopWords()[:-1])
        if isinstance(pipeline, Pipeline):
            pipeline.setStages(stages)
        else:
            pipeline.stages = stages
        return pipeline


class _CarrierWriter(MLWriter):
    def saveImpl(self, path: str) -> None:
        self.instance._to_java()._save_impl(path)


class PysparkReaderWriter(object):
    """Mixin: ``write()/save()`` persist the stage as a carrier; ``read()/load()`` restore it.  With a genuine PySpark the
    carrier is a JVM ``StopWordsRemover`` written by ``JavaMLWriter`` (what the reference does); without one the
    stand-in writes the same directory layout itself."""

    def write(self):
        if REAL_PYSPARK:
            return JavaMLWriter(self)
        return _CarrierWriter(self)

    def save(self, path: str) -> None:
        self.write().save(path)

    @classmethod
    def read(cls):
        if REAL_PYSPARK:
            return JavaMLReader(PysparkObjId._getCarrierClass())
        return MLReader(PysparkObjId._getCarrierClass())

    @classmethod
    def load(cls, path: str):
        return cls._from_java(cls.read().load(path))

    @classmethod
    def _from_java(cls, java_obj):
        return load_byte_array(list(java_obj.getStopWords())[:-1])

    def _to_java(self):
        if REAL_PYSPARK:
            # a JVM StopWordsRemover carrying this object's uid, its stop words = [payload, GUID]
            from pyspark import SparkContext
            from pyspark.ml.wrapper import JavaParams

            words = dump_byte_array(self) + [PysparkObjId._getPyObjId()]
            gateway = SparkContext._active_spark_context._gateway
            jwords = gateway.new_array(gateway.jvm.java.lang.String, len(words))
            for i, w in enumerate(words):
                jwords[i] = w
            jcarrier = JavaParams._new_java_obj(PysparkObjId._getCarrierClass(javaName=True), self.uid)
            jcarrier.setStopWords(jwords)
            return jcarrier
        carrier = StopWordsRemover()
        carrier._resetUid(self.uid)
        carrier.setStopWords(dump_byte_array(self) + [PysparkObjId._getPyObjId()])
        return carrier
