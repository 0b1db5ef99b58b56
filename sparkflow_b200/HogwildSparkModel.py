"""``HogwildSparkModel``: asynchronous parameter-server training over the partitions of an RDD.

Public API parity with lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:103-272 (constructor keywords,
``train(rdd) -> list of numpy weights``, ``stop_server()``, ``determine_master``, module-level
``get_server_weights`` / ``put_deltas_to_server``), with the Flask/HTTP/pickle machinery replaced by
:class:`sparkflow_b200.parallel.session.TrainingSession` (fused NVLink push/pull kernels on H100,
threads or gloo on CPU).  ``serverStartup`` is accepted and ignored: readiness is explicit, there is
no start-up sleep.
"""
from __future__ import annotations

import random
import socket
from typing import Callable, Dict, List, Optional

import numpy as np

from .ml_util import handle_features
from .ops.optimizers import OptimizerSpec
from .parallel import dist as D
from .parallel.session import TrainingSession
from .spark.backend import collect_partitions

# live sessions by master url, so the module-level helper functions of the reference keep working
_SERVERS: Dict[str, "HogwildSparkModel"] = {}


def get_server_weights(master_url: str = "localhost:5000") -> List[np.ndarray]:
    """Current master weights (reference: HTTP GET /parameters, HogwildSparkModel.py:22-28)."""
    model = _SERVERS.get(master_url) or _SERVERS.get(_port_key(master_url))
    if model is None:
        raise ConnectionError(f"no parameter server is running at {master_url}")
    return model._session.weights()


def put_deltas_to_server(delta, master_url: str = "localhost:5000") -> None:
    """Apply one gradient list as ONE optimizer step on the master (reference: HTTP POST /update)."""
    model = _SERVERS.get(master_url) or _SERVERS.get(_port_key(master_url))
    if model is None:
        raise ConnectionError(f"no parameter server is running at {master_url}")
    model._session.push_external(delta)


def _port_key(url: str) -> str:
    return ":" + url.rsplit(":", 1)[-1]


def handle_model(data, graph_json, tfInput, tfLabel=None, master_url="localhost:5000", iters=1000, mini_batch_size=-1, shuffle=True,
                 mini_stochastic_iters=-1, verbose=0, loss_callback=None):
    """The per-partition worker body (reference: HogwildSparkModel.py:38-100, the function shipped to
    ``rdd.foreachPartition``): train on the rows of ONE partition against the parameter server registered at
    ``master_url`` with the reference's loop semantics (modes A / B / C, ``n - 1`` clamp, per-iteration shuffle,
    ``verbose`` print format, ``loss_callback(loss, iteration, partition_id)``).  ``graph_json`` must be the graph the
    server was started with.  Returns the partition id."""
    from .parallel.worker import run_partition

    model = _SERVERS.get(master_url) or _SERVERS.get(_port_key(master_url))
    if model is None:
        raise ConnectionError(f"no parameter server is running at {master_url}")
    sess = model._session
    if graph_json is not None and graph_json != sess.graph_json:
        raise ValueError("handle_model: graph_json differs from the graph the parameter server at %s was started with" % master_url)
    features, labels = handle_features(data, tfLabel is not None)
    if features.shape[0] == 0:
        return None
    engine = sess.make_engine(sess.local_devices()[0] if sess.use_cuda else __import__("torch").device("cpu"))
    return run_partition(engine, features, labels, iters=iters, mini_batch_size=mini_batch_size, shuffle=shuffle,
                         mini_stochastic_iters=mini_stochastic_iters, verbose=verbose, loss_callback=loss_callback)


class HogwildSparkModel(object):
    """Hogwild! / locked asynchronous SGD: every partition is a worker that pulls the master
    parameters, computes a gradient on a minibatch and pushes it; the master applies one optimizer
    step per push without aggregating across workers."""

    def __init__(self, tensorflowGraph=None, iters=1000, tfInput=None, tfLabel=None, optimizer=None, master_url=None,
                 serverStartup=8, acquire_lock=False, mini_batch=-1, mini_stochastic_iters=-1, shuffle=True, verbose=0,
                 partition_shuffles=1, loss_callback: Optional[Callable] = None, port=5000, engine="auto", seed=None,
                 initial_weights=None, resume_from=None, checkpoint_dir=None, checkpoint_every=0):
        self.tensorflowGraph = tensorflowGraph
        self.iters = iters
        self.tfInput = tfInput
        self.tfLabel = tfLabel
        self.acquire_lock = acquire_lock
        self.mini_batch = mini_batch
        self.mini_stochastic_iters = mini_stochastic_iters
        self.verbose = verbose
        self.shuffle = shuffle
        self.partition_shuffles = partition_shuffles
        self.loss_callback = loss_callback
        self.port = port
        self.master_url = master_url if master_url is not None else HogwildSparkModel.determine_master(port)
        if optimizer is None:
            optimizer = OptimizerSpec.from_tf_kwargs("gradient_descent", {"learning_rate": 0.01})
        if not isinstance(optimizer, OptimizerSpec):
            raise TypeError("optimizer must come from build_optimizer(...) or tf.train.*Optimizer of sparkflow_b200's tf shim")
        self.optimizer = optimizer
        self._session = TrainingSession(tensorflowGraph, tfInput, tfLabel, optimizer, acquire_lock=acquire_lock, iters=iters,
                                        mini_batch=mini_batch, mini_stochastic_iters=mini_stochastic_iters, shuffle=shuffle,
                                        verbose=verbose, loss_callback=loss_callback, engine=engine, seed=seed,
                                        initial_weights=initial_weights, resume_from=resume_from, checkpoint_dir=checkpoint_dir,
                                        checkpoint_every=checkpoint_every)
        self.start_server()

    @staticmethod
    def determine_master(port):
        try:
            return socket.gethostbyname(socket.gethostname()) + ":" + str(port)
        except Exception:
            return "localhost:" + str(port)

    def start_server(self, *_ignored):
        """Bring the master state up (synchronously; returns when it is ready to serve)."""
        self._session.open()
        _SERVERS[self.master_url] = self
        _SERVERS[_port_key(self.master_url)] = self
        self.server = self._session

    def start_service(self, metagraph=None, optimizer=None, port=None):
        """Reference: the body of the Flask process (HogwildSparkModel.py:175-244).  There is no separate service
        process here - the master state lives on the driver GPU (or in this process on CPU) - so this is
        ``start_server`` under the reference's name; ``metagraph`` / ``optimizer`` / ``port`` must be the ones the model
        was constructed with and are only checked."""
        if metagraph is not None and metagraph != self.tensorflowGraph:
            raise ValueError("start_service: a different graph than the one this model was built with")
        if port is not None and int(port) != int(self.port):
            raise ValueError("start_service: a different port than the one this model was built with")
        self.start_server()

    def stop_server(self):
        """Release the master state. Idempotent."""
        for k in [k for k, v in _SERVERS.items() if v is self]:
            _SERVERS.pop(k, None)
        self._session.close()

    def train(self, rdd):
        """Run ``partition_shuffles`` rounds of ``iters`` iterations over every partition and return
        the final master weights as a list of numpy arrays (trainable-variable order)."""
        try:
            supervised = self.tfLabel is not None
            ctx = self._session.ctx
            for rnd in range(self.partition_shuffles):
                parts = [handle_features(iter(p), supervised) for p in collect_partitions(rdd)]
                parts = [(f, l) for f, l in parts if f.shape[0] > 0]
                self._session.train_partitions(parts)
                if self.partition_shuffles - rnd > 1:
                    seed = D.broadcast_object(ctx, random.randrange(1 << 30), src=0)
                    state = random.getstate()
                    random.seed(seed)                      # identical repartition on every rank
                    rdd = rdd.repartition(rdd.getNumPartitions())
                    random.setstate(state)
            weights = self._session.weights()
            self.stop_server()
            return weights
        except Exception:
            self.stop_server()
            raise
