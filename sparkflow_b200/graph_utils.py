"""``build_graph`` and the optimizer-config builders.

API parity with lifeomic/sparkflow/sparkflow/graph_utils.py (build_graph :6-15, config builders :18-47).
``build_graph(func)`` runs ``func`` inside a fresh graph and returns the MetaGraphDef as proto3 JSON.
With real TensorFlow 1.x importable, its ``tf.Graph``/``export_meta_graph`` are used; otherwise the
built-in TF-compatible builder (``sparkflow_b200.graph.tfcompat``) produces the same JSON layout.
"""
from __future__ import annotations

import json
from typing import Callable


def _tf():
    try:  # pragma: no cover - TensorFlow 1.x is not installable in this image
        import tensorflow as real_tf

        if hasattr(real_tf, "train") and hasattr(real_tf.train, "export_meta_graph") and not getattr(real_tf, "_sparkflow_shim", False):
            return real_tf, True
    except Exception:
        pass
    from .graph import tfcompat

    return tfcompat, False


def build_graph(func: Callable[[], object]) -> str:
    """:param func: function that builds the model (placeholders, layers, a ``tf.losses`` loss)
    :return: MetaGraphDef of the graph ``func`` built, as a JSON string"""
    tf, is_real = _tf()
    graph = tf.Graph()
    with graph.as_default():
        func()
        mg = tf.train.export_meta_graph()
    if is_real:  # pragma: no cover
        from google.protobuf import json_format

        return json_format.MessageToJson(mg)
    return mg.to_json()


def generate_config(**kwargs) -> str:
    return json.dumps(kwargs)


def _config(locals_: dict) -> str:
    return generate_config(**{k: v for k, v in locals_.items()})


def build_adam_config(learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, use_locking=False) -> str:
    return _config(locals())


def build_rmsprop_config(learning_rate=0.001, decay=0.9, momentum=0.0, epsilon=1e-10, use_locking=False, centered=False) -> str:
    return _config(locals())


def build_momentum_config(learning_rate=0.001, momentum=0.9, use_locking=False, use_nesterov=False) -> str:
    return _config(locals())


def build_adadelta_config(learning_rate=0.001, rho=0.95, epsilon=1e-8, use_locking=False) -> str:
    return _config(locals())


def build_adagrad_config(learning_rate=0.001, initial_accumulator=0.1, use_locking=False) -> str:
    # the reference emits the key ``initial_accumulator`` (graph_utils.py:42); TF's own keyword is
    # ``initial_accumulator_value`` – the optimizer factory here accepts both spellings.
    return _config(locals())


def build_gradient_descent(learning_rate=0.001, use_locking=False) -> str:
    return _config(locals())


def build_ftrl_config(learning_rate=0.001, learning_rate_power=-0.5, initial_accumulator_value=0.1,
                      l1_regularization_strength=0.0, l2_regularization_strength=0.0, use_locking=False) -> str:
    return _config(locals())


def build_proximal_adagrad_config(learning_rate=0.001, initial_accumulator_value=0.1, l1_regularization_strength=0.0,
                                  l2_regularization_strength=0.0, use_locking=False) -> str:
    return _config(locals())


def build_proximal_gradient_descent_config(learning_rate=0.001, l1_regularization_strength=0.0,
                                           l2_regularization_strength=0.0, use_locking=False) -> str:
    return _config(locals())


def build_adagrad_da_config(learning_rate=0.001, initial_gradient_squared_accumulator_value=0.1,
                            l1_regularization_strength=0.0, l2_regularization_strength=0.0, use_locking=False) -> str:
    return _config(locals())
