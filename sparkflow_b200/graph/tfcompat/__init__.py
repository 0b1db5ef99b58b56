"""``import sparkflow_b200.graph.tfcompat as tf`` – the TF-1.x graph-construction API subset that
lifeomic/sparkflow user code relies on (README.md:39-47, examples/*.py, tests/dl_runner.py:45-73),
implemented without TensorFlow.  ``sparkflow_b200.compat.install()`` registers it as ``tensorflow``
when the real package is absent so reference scripts run unchanged.
"""
from __future__ import annotations

import types as _types

from . import core as _core
from . import ops as _ops
from . import train as _train_mod
from .core import (DType, Graph, GraphKeys, MetaGraphDef, Operation, Tensor, TensorShape, Variable as _Var, as_dtype,  # noqa: F401
                   bool_ as bool, convert_to_tensor, float16, float32, float64, get_default_graph, int32, int64,  # noqa: A004
                   reset_default_graph, uint8)
from .ops import (abs, add, argmax, cast, concat, constant, constant_initializer, divide, exp, expand_dims,  # noqa: A004,F401
                  get_variable, global_variables, global_variables_initializer, glorot_normal_initializer,
                  glorot_uniform_initializer, identity, log, matmul, maximum, minimum, multiply, negative,
                  ones_initializer, placeholder, placeholder_with_default, pow, random_normal_initializer,  # noqa: A004
                  random_uniform_initializer, reduce_max, reduce_mean, reduce_sum, reshape, shape, sigmoid, size, sqrt,
                  square, squared_difference, squeeze, stop_gradient, subtract, tanh, trainable_variables, transpose,
                  truncated_normal_initializer, zeros_initializer)
from .ops import (ceil, clip_by_value, equal, floor, greater, greater_equal, less, less_equal, log1p, logical_and,  # noqa: F401
                  logical_not, not_equal, ones_like, reciprocal, reduce_min, reduce_prod, rsqrt, sign, stack, tile, where,
                  zeros_like)
from .ops import (cond, cos, cumsum, erf, floormod, gather, logical_or, one_hot, pad, reduce_all, reduce_any, round, sin, split,  # noqa: A004,F401
                  unstack)
from .ops import add_n  # noqa: F401
from .session import InteractiveSession, Session, get_default_session  # noqa: F401

__version__ = "1.10.0-sparkflow_b200"
VERSION = __version__
double = float64
half = float16


def Variable(initial_value=None, trainable=True, name=None, dtype=None, **kw):  # noqa: N802
    return _ops.variable(initial_value, trainable=trainable, name=name, dtype=dtype, **kw)


def name_scope(name, default_name=None, values=None):
    return get_default_graph().name_scope(name or default_name)


def variable_scope(name_or_scope, default_name=None, reuse=None, **_unused):
    return get_default_graph().name_scope(name_or_scope or default_name)


def get_collection(key, scope=None):
    return get_default_graph().get_collection(key, scope)


def add_to_collection(name, value):
    get_default_graph().add_to_collection(name, value)


def set_random_seed(seed):
    get_default_graph().seed = seed


def gradients(ys, xs, **_unused):
    raise NotImplementedError("tf.gradients is provided by the engine (autograd / hand-written backward kernels); "
                              "graphs only need to register their loss in the 'losses' collection")


truediv = div = divide
sub = subtract
mul = multiply
neg = negative
to_float = lambda x, name="ToFloat": cast(x, float32, name)  # noqa: E731
arg_max = argmax
mod = floormod

nn = _types.SimpleNamespace(
    relu=_ops.relu, sigmoid=_ops.sigmoid, tanh=_ops.tanh, softmax=_ops.softmax, softplus=_ops.softplus, elu=_ops.elu,
    leaky_relu=_ops.leaky_relu, bias_add=_ops.bias_add, conv2d=_ops.conv2d, max_pool=_ops.max_pool, avg_pool=_ops.avg_pool,
    dropout=_ops.dropout, softmax_cross_entropy_with_logits=_ops.softmax_cross_entropy_with_logits,
    softmax_cross_entropy_with_logits_v2=_ops.softmax_cross_entropy_with_logits,
    sigmoid_cross_entropy_with_logits=_ops.sigmoid_cross_entropy_with_logits,
    relu6=_ops.relu6, selu=_ops.selu, softsign=_ops.softsign, log_softmax=_ops.log_softmax, l2_loss=_ops.l2_loss,
    l2_normalize=_ops.l2_normalize, embedding_lookup=_ops.embedding_lookup,
    sparse_softmax_cross_entropy_with_logits=_ops.sparse_softmax_cross_entropy_with_logits, conv2d_transpose=_ops.conv2d_transpose,
    depthwise_conv2d=_ops.depthwise_conv2d, top_k=_ops.top_k,
)
layers = _types.SimpleNamespace(
    dense=_ops.dense, conv2d=_ops.conv2d_layer, max_pooling2d=_ops.max_pooling2d, average_pooling2d=_ops.average_pooling2d,
    flatten=_ops.flatten, dropout=_ops.dropout_layer, batch_normalization=_ops.batch_normalization,
    conv2d_transpose=_ops.conv2d_transpose_layer,
)
losses = _types.SimpleNamespace(
    softmax_cross_entropy=_ops.softmax_cross_entropy, mean_squared_error=_ops.mean_squared_error,
    sigmoid_cross_entropy=_ops.sigmoid_cross_entropy, absolute_difference=_ops.absolute_difference,
    add_loss=_ops.add_loss, get_losses=_ops.get_losses, log_loss=_ops.log_loss, hinge_loss=_ops.hinge_loss,
    huber_loss=_ops.huber_loss, sparse_softmax_cross_entropy=_ops.sparse_softmax_cross_entropy,
    get_regularization_loss=_ops.get_regularization_loss,
)
initializers = _types.SimpleNamespace(
    glorot_uniform=glorot_uniform_initializer, glorot_normal=glorot_normal_initializer, zeros=zeros_initializer,
    ones=ones_initializer, constant=constant_initializer, random_uniform=random_uniform_initializer,
    random_normal=random_normal_initializer, truncated_normal=truncated_normal_initializer,
)
contrib = _types.SimpleNamespace(layers=_types.SimpleNamespace(
    xavier_initializer=lambda uniform=True, seed=None, dtype=float32: (glorot_uniform_initializer(seed) if uniform else glorot_normal_initializer(seed)),
    fully_connected=lambda inputs, num_outputs, activation_fn=_ops.relu, **kw: _ops.dense(inputs, num_outputs, activation=activation_fn, **kw),
    flatten=_ops.flatten, l2_regularizer=_ops.l2_regularizer,
))
train = _train_mod
keras = _types.SimpleNamespace(initializers=initializers)
