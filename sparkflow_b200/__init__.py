"""sparkflow_b200 – a Hopper-native asynchronous parameter-server training framework with the
public API of lifeomic/sparkflow (SparkAsyncDL / SparkAsyncDLModel / HogwildSparkModel / build_graph /
PysparkPipelineWrapper / load_tensorflow_model) and its artefact formats.

Layout
------
``graph/``     TF-compatible graph builder, MetaGraphDef codec, IR, PyTorch interpreter (oracle / CPU)
``models/``    graph -> layer-plan compiler and the model zoo
``ops/``       native-extension loader, flat parameter layout, optimizer rules
``parallel/``  H100 device engine, host parameter server (threads / gloo), worker loop, sessions
``spark/``     dependency-free stand-in for the used slice of PySpark (DataFrame, ML Pipeline, persistence)
``io/``        TF-V2 checkpoint bundles, CSV
``utils/``     timing, clocks, tracing, metrics, fault injection
``csrc/``      (repo root) sm_90a kernels + C++ runtime
"""
__version__ = "0.2.0"

import os as _os

# Single-process multi-worker runs (several worker threads + shard appliers on the same GPU, e.g. the test-suite) create
# more streams than the default 8 hardware launch queues; streams that share a queue can delay each other's launches.
# Opt in with SPARKFLOW_MAX_CONNECTIONS=32 (must be set before the CUDA context exists); one-process-per-GPU runs use 7
# streams and keep the driver default.
if _os.environ.get("SPARKFLOW_MAX_CONNECTIONS"):
    _os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", _os.environ["SPARKFLOW_MAX_CONNECTIONS"])

from .graph_utils import (build_adadelta_config, build_adagrad_config, build_adam_config, build_gradient_descent,  # noqa: F401
                          build_graph, build_momentum_config, build_rmsprop_config)
