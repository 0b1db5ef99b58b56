"""Model zoo: every workload the reference ships (SURVEY.md section 2.3) plus the BASELINE.json
stress configs, as plain graph-builder functions usable with ``build_graph``.

Each function mirrors a model definition of the reference:
  * :func:`simple_dnn`        – examples/simple_dnn.py:13-21 (784-256-256-10, softmax-CE, ``out`` = argmax)
  * :func:`cnn`               – examples/cnn_example.py:10-22 (conv5x5x32-pool-conv3x3x64-pool-dense10)
  * :func:`autoencoder`       – examples/autoencoder_example.py:9-16 (784-256-128-256-784, MSE vs input)
  * :func:`test_mlp` / :func:`test_autoencoder` – tests/dl_runner.py:45-73
  * :func:`fixture_mlp`       – the graph stored in tests/test_model/to_load.meta (2-10-10-1)
  * :func:`autoencoder_small` / :func:`wide_dnn` – BASELINE.json configs 4 and 5
  * :func:`cnn_same`          – TensorFlow's "Deep MNIST" network (SAME-padded convs and pools)
  * :func:`cnn_strided`       – strided / SAME convs, a conv feeding a conv, an overlapping 3x3/2 pool, a conv feeding
    the flatten
  * :func:`binary_dnn` / :func:`multilabel_dnn` – binary and multi-label classifiers trained with sigmoid cross-entropy
  * :func:`selu_dnn` / :func:`leaky_cnn` / :func:`softplus_autoencoder` – SELU, leaky ReLU + ELU and softplus networks
  * :func:`sparse_dnn` / :func:`onehot_cnn` / :func:`sparse_dnn100` – classifiers trained on a numeric class column
    ([None, 1] labels) with sparse softmax cross-entropy or a ``tf.one_hot`` in the graph
  * :func:`l2_dnn` / :func:`l2_cnn` / :func:`l2_autoencoder` – simple_dnn, cnn_same and autoencoder with an L2 weight
    penalty in the loss, in three TF-1.x spellings
  * :func:`dropout_cnn` / :func:`conv_dropout_cnn` – the Keras MNIST CNN (dropout after the pool and after the hidden dense
    layer) and dropouts on conv outputs, a general pool and a flatten
"""
from __future__ import annotations

from typing import Callable, Dict

from ..graph import tfcompat as tf


def simple_dnn():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    h1 = tf.layers.dense(x, 256, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    h2 = tf.layers.dense(h1, 256, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    logits = tf.layers.dense(h2, 10, kernel_initializer=tf.glorot_uniform_initializer())
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def binary_dnn():
    """784-256-256-1 binary classifier: sigmoid cross-entropy on the logit, ``out`` = its probability"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    h1 = tf.layers.dense(x, 256, activation=tf.nn.relu)
    h2 = tf.layers.dense(h1, 256, activation=tf.nn.relu)
    logits = tf.layers.dense(h2, 1)
    tf.nn.sigmoid(logits, name="out")
    return tf.losses.sigmoid_cross_entropy(y, logits)


def multilabel_dnn(tags: int = 40):
    """784-256-``tags`` multi-label classifier: one independent sigmoid cross-entropy per tag, spelled as
    ``reduce_mean(sigmoid_cross_entropy_with_logits)`` + ``add_loss``"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, tags], name="y")
    h = tf.layers.dense(x, 256, activation=tf.nn.relu)
    logits = tf.layers.dense(h, tags)
    tf.nn.sigmoid(logits, name="out")
    loss = tf.reduce_mean(tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits))
    tf.losses.add_loss(loss)
    return loss


def sparse_dnn():
    """simple_dnn trained on a numeric class column (e.g. StringIndexer output): a [None, 1] label placeholder and
    ``tf.losses.sparse_softmax_cross_entropy``"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    h1 = tf.layers.dense(x, 256, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    h2 = tf.layers.dense(h1, 256, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    logits = tf.layers.dense(h2, 10, kernel_initializer=tf.glorot_uniform_initializer())
    tf.argmax(logits, 1, name="out")
    return tf.losses.sparse_softmax_cross_entropy(tf.cast(tf.reshape(y, [-1]), tf.int32), logits)


def sparse_dnn100():
    """784-256-100 classifier on class indices, spelled ``reduce_mean(sparse_softmax_cross_entropy_with_logits)`` +
    ``add_loss`` (100 classes: wider than the fused softmax head)"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    h = tf.layers.dense(x, 256, activation=tf.nn.relu)
    logits = tf.layers.dense(h, 100)
    tf.argmax(logits, 1, name="out")
    loss = tf.reduce_mean(tf.nn.sparse_softmax_cross_entropy_with_logits(labels=tf.cast(tf.squeeze(y, axis=1), tf.int64),
                                                                         logits=logits))
    tf.losses.add_loss(loss)
    return loss


def cnn():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.max_pooling2d(tf.layers.conv2d(img, 32, 5, activation=tf.nn.relu), 2, 2)
    c2 = tf.layers.max_pooling2d(tf.layers.conv2d(c1, 64, 3, activation=tf.nn.relu), 2, 2)
    logits = tf.layers.dense(tf.layers.flatten(c2), 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def onehot_cnn():
    """cnn on a numeric class column, one-hot encoded in the graph: ``tf.one_hot`` of the [None, 1] label column"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.max_pooling2d(tf.layers.conv2d(img, 32, 5, activation=tf.nn.relu), 2, 2)
    c2 = tf.layers.max_pooling2d(tf.layers.conv2d(c1, 64, 3, activation=tf.nn.relu), 2, 2)
    logits = tf.layers.dense(tf.layers.flatten(c2), 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(tf.one_hot(tf.cast(tf.reshape(y, [-1]), tf.int32), 10), logits)


def cnn_same():
    """conv 5x5x32 SAME relu -> pool 2x2/2 SAME -> conv 5x5x64 SAME relu -> pool 2x2/2 SAME -> dense 1024 relu -> dense 10"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.max_pooling2d(tf.layers.conv2d(img, 32, 5, padding="same", activation=tf.nn.relu), 2, 2, padding="same")
    c2 = tf.layers.max_pooling2d(tf.layers.conv2d(c1, 64, 5, padding="same", activation=tf.nn.relu), 2, 2, padding="same")
    h = tf.layers.dense(tf.layers.flatten(c2), 1024, activation=tf.nn.relu)
    logits = tf.layers.dense(h, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def cnn_strided():
    """28x28x1 -> conv 3x3x16 SAME relu -> conv 3x3x32 SAME stride 2 tanh -> pool 3x3/2 SAME -> conv 3x3x32 VALID stride 2 relu
    -> flatten 288 -> dense 10"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.conv2d(img, 16, 3, padding="same", activation=tf.nn.relu)
    c2 = tf.layers.conv2d(c1, 32, 3, strides=2, padding="same", activation=tf.nn.tanh)
    p2 = tf.layers.max_pooling2d(c2, 3, 2, padding="same")
    c3 = tf.layers.conv2d(p2, 32, 3, strides=2, padding="valid", activation=tf.nn.relu)
    logits = tf.layers.dense(tf.layers.flatten(c3), 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def selu_dnn():
    """784-256-256-10 self-normalising classifier: SELU hidden layers, softmax-CE"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    h1 = tf.layers.dense(x, 256, activation=tf.nn.selu)
    h2 = tf.layers.dense(h1, 256, activation=tf.nn.selu)
    logits = tf.layers.dense(h2, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def leaky_cnn():
    """cnn_same with leaky ReLU (alpha 0.1) convs and an ELU dense layer"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])

    def leaky(t):
        return tf.nn.leaky_relu(t, alpha=0.1)

    c1 = tf.layers.max_pooling2d(tf.layers.conv2d(img, 32, 5, padding="same", activation=leaky), 2, 2, padding="same")
    c2 = tf.layers.max_pooling2d(tf.layers.conv2d(c1, 64, 5, padding="same", activation=leaky), 2, 2, padding="same")
    h = tf.layers.dense(tf.layers.flatten(c2), 1024, activation=tf.nn.elu)
    logits = tf.layers.dense(h, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def softplus_autoencoder():
    """784-128-784 auto-encoder: softplus code, sigmoid reconstruction, MSE against the input"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    code = tf.layers.dense(x, 128, activation=tf.nn.softplus, name="out")
    rec = tf.layers.dense(code, 784, activation=tf.nn.sigmoid)
    return tf.losses.mean_squared_error(rec, x)


def autoencoder():
    x = tf.placeholder("float", shape=[None, 784], name="x")
    e1 = tf.layers.dense(x, 256, activation=tf.nn.relu)
    code = tf.layers.dense(e1, 128, activation=tf.nn.sigmoid, name="out")
    d1 = tf.layers.dense(code, 256, activation=tf.nn.relu)
    rec = tf.layers.dense(d1, 784, activation=tf.nn.sigmoid)
    return tf.losses.mean_squared_error(rec, x)


def autoencoder_small():
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    code = tf.layers.dense(x, 32, activation=tf.nn.sigmoid, name="out")
    rec = tf.layers.dense(code, 784, activation=tf.nn.sigmoid)
    return tf.losses.mean_squared_error(rec, x)


def wide_dnn(width: int = 4096, depth: int = 4, classes: int = 1000):
    x = tf.placeholder(tf.float32, shape=[None, width], name="x")
    y = tf.placeholder(tf.float32, shape=[None, classes], name="y")
    h = x
    for _ in range(depth):
        h = tf.layers.dense(h, width, activation=tf.nn.relu)
    logits = tf.layers.dense(h, classes)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def l2_dnn():
    """simple_dnn with ``5e-4 * add_n(l2_loss)`` of its three kernels added to the loss"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    h1 = tf.layers.dense(x, 256, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    h2 = tf.layers.dense(h1, 256, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    logits = tf.layers.dense(h2, 10, kernel_initializer=tf.glorot_uniform_initializer())
    tf.argmax(logits, 1, name="out")
    kernels = [v for v in tf.trainable_variables() if v.name.split(":")[0].endswith("/kernel")]
    loss = (tf.reduce_mean(tf.nn.softmax_cross_entropy_with_logits(labels=y, logits=logits))
            + 5e-4 * tf.add_n([tf.nn.l2_loss(w) for w in kernels]))
    tf.losses.add_loss(loss)
    return loss


def l2_cnn():
    """cnn_same with ``l2_regularizer(1e-4)`` kernel regularizers: ``softmax_cross_entropy`` outside the losses
    collection plus ``get_regularization_loss()``, added with ``add_loss``"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    reg = tf.contrib.layers.l2_regularizer(1e-4)
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.max_pooling2d(tf.layers.conv2d(img, 32, 5, padding="same", activation=tf.nn.relu, kernel_regularizer=reg), 2, 2,
                                 padding="same")
    c2 = tf.layers.max_pooling2d(tf.layers.conv2d(c1, 64, 5, padding="same", activation=tf.nn.relu, kernel_regularizer=reg), 2, 2,
                                 padding="same")
    h = tf.layers.dense(tf.layers.flatten(c2), 1024, activation=tf.nn.relu, kernel_regularizer=reg)
    logits = tf.layers.dense(h, 10, kernel_regularizer=reg)
    tf.argmax(logits, 1, name="out")
    loss = tf.losses.softmax_cross_entropy(y, logits, loss_collection=None) + tf.losses.get_regularization_loss()
    tf.losses.add_loss(loss)
    return loss


def l2_autoencoder():
    """autoencoder with ``1e-5 * add_n(l2_loss)`` of every trainable variable, biases included"""
    x = tf.placeholder("float", shape=[None, 784], name="x")
    e1 = tf.layers.dense(x, 256, activation=tf.nn.relu)
    code = tf.layers.dense(e1, 128, activation=tf.nn.sigmoid, name="out")
    d1 = tf.layers.dense(code, 256, activation=tf.nn.relu)
    rec = tf.layers.dense(d1, 784, activation=tf.nn.sigmoid)
    loss = (tf.losses.mean_squared_error(rec, x, loss_collection=None)
            + 1e-5 * tf.add_n([tf.nn.l2_loss(v) for v in tf.trainable_variables()]))
    tf.losses.add_loss(loss)
    return loss


def dropout_cnn():
    """The Keras MNIST CNN: conv 3x3x32 VALID relu -> conv 3x3x64 VALID relu -> pool 2x2/2 -> dropout 0.25 -> flatten ->
    dense 128 relu -> dropout 0.5 -> dense 10"""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c1 = tf.layers.conv2d(img, 32, 3, activation=tf.nn.relu)
    c2 = tf.layers.conv2d(c1, 64, 3, activation=tf.nn.relu)
    p = tf.layers.dropout(tf.layers.max_pooling2d(c2, 2, 2), rate=0.25, training=True)
    h = tf.layers.dropout(tf.layers.dense(tf.layers.flatten(p), 128, activation=tf.nn.relu), rate=0.5, training=True)
    logits = tf.layers.dense(h, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def conv_dropout_cnn():
    """28x28x1 -> conv 3x3x16 SAME relu -> pool 2x2/2 -> dropout 0.9 -> conv 3x3x32 SAME tanh -> dropout 0.8 (keep_prob
    placeholder with a default) -> pool 3x3/2 SAME -> conv 3x3x32 VALID relu -> dropout 0.75 -> conv 3x3x16 SAME sigmoid ->
    flatten -> dropout 0.6 -> dense 10.  The first conv + pool carries a dropout, so it runs as im2col + GEMM."""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    kp = tf.placeholder_with_default(0.8, shape=[], name="keep_prob")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    p1 = tf.nn.dropout(tf.layers.max_pooling2d(tf.layers.conv2d(img, 16, 3, padding="same", activation=tf.nn.relu), 2, 2), keep_prob=0.9)
    c2 = tf.nn.dropout(tf.layers.conv2d(p1, 32, 3, padding="same", activation=tf.nn.tanh), keep_prob=kp)
    p2 = tf.layers.max_pooling2d(c2, 3, 2, padding="same")
    c3 = tf.nn.dropout(tf.layers.conv2d(p2, 32, 3, activation=tf.nn.relu), keep_prob=0.75)
    c4 = tf.layers.conv2d(c3, 16, 3, padding="same", activation=tf.nn.sigmoid)
    logits = tf.layers.dense(tf.nn.dropout(tf.layers.flatten(c4), keep_prob=0.6), 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def test_mlp(in_dim: int = 10):
    x = tf.placeholder(tf.float32, shape=[None, in_dim], name="x")
    h1 = tf.layers.dense(x, 12, activation=tf.nn.relu)
    h2 = tf.layers.dense(h1, 7, activation=tf.nn.relu)
    out = tf.layers.dense(h2, 1, name="outer", activation=tf.nn.sigmoid)
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    return tf.losses.mean_squared_error(y, out)


def test_autoencoder():
    x = tf.placeholder(tf.float32, shape=[None, 10], name="x")
    enc = tf.layers.dense(x, 5, activation=tf.nn.relu)
    code = tf.layers.dense(enc, 2, activation=tf.nn.sigmoid, name="out")
    dec = tf.layers.dense(code, 5, activation=tf.nn.relu)
    rec = tf.layers.dense(dec, 10)
    return tf.losses.mean_squared_error(x, rec)


def fixture_mlp():
    x = tf.placeholder(tf.float32, shape=[None, 2], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    h1 = tf.layers.dense(x, 10, activation=tf.nn.tanh)
    h2 = tf.layers.dense(h1, 10, activation=tf.nn.tanh)
    out = tf.layers.dense(h2, 1, activation=tf.nn.sigmoid, name="out")
    return tf.losses.mean_squared_error(y, out)


MODELS: Dict[str, Callable] = {
    "simple_dnn": simple_dnn,
    "cnn": cnn,
    "cnn_same": cnn_same,
    "cnn_strided": cnn_strided,
    "autoencoder": autoencoder,
    "autoencoder_small": autoencoder_small,
    "wide_dnn": wide_dnn,
    "test_mlp": test_mlp,
    "test_autoencoder": test_autoencoder,
    "fixture_mlp": fixture_mlp,
    "binary_dnn": binary_dnn,
    "multilabel_dnn": multilabel_dnn,
    "selu_dnn": selu_dnn,
    "leaky_cnn": leaky_cnn,
    "softplus_autoencoder": softplus_autoencoder,
    "sparse_dnn": sparse_dnn,
    "onehot_cnn": onehot_cnn,
    "sparse_dnn100": sparse_dnn100,
    "l2_dnn": l2_dnn,
    "l2_cnn": l2_cnn,
    "l2_autoencoder": l2_autoencoder,
    "dropout_cnn": dropout_cnn,
    "conv_dropout_cnn": conv_dropout_cnn,
}


def build(name: str, **kwargs) -> str:
    """MetaGraphDef JSON of a zoo model (same as ``build_graph(MODELS[name])``)."""
    g = tf.Graph()
    with g.as_default():
        MODELS[name](**kwargs)
        return tf.train.export_meta_graph().to_json(indent=None)
