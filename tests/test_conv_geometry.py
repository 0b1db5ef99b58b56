"""Compiled-plan geometry of SAME-padded / strided convolutions and general max-pools (no GPU): the compiler's layer
shapes, strides and pads against hand-computed TensorFlow numbers, and what the plan grammar accepts and rejects."""
import pytest

from sparkflow_b200.graph import tfcompat as tf
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.graph_utils import build_graph
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import UnsupportedGraph, compile_graph, conv_geometry
from sparkflow_b200.parallel.plan_builder import check_grammar, fused_first_conv


def _plan(name):
    return compile_graph(GraphIR.from_metagraph(zoo.build(name)), "x:0", "y:0")


def _geo(lp):
    return [(l.kind, l.in_shape, l.out_shape, l.ksize, l.strides, l.pads) for l in lp.layers if l.kind in ("conv", "pool")]


def test_cnn_same_layers():
    lp = _plan("cnn_same")
    assert [l.kind for l in lp.layers] == ["reshape", "conv", "pool", "conv", "pool", "reshape", "dense", "dense"]
    assert _geo(lp) == [
        ("conv", (28, 28, 1), (28, 28, 32), (5, 5), (1, 1), (2, 2, 2, 2)),
        ("pool", (28, 28, 32), (14, 14, 32), (2, 2), (2, 2), (0, 0, 0, 0)),      # SAME 2x2/2 on an even size: no padding
        ("conv", (14, 14, 32), (14, 14, 64), (5, 5), (1, 1), (2, 2, 2, 2)),
        ("pool", (14, 14, 64), (7, 7, 64), (2, 2), (2, 2), (0, 0, 0, 0)),
    ]
    assert lp.layers[6].in_shape == (3136,) and lp.layers[6].out_shape == (1024,)
    check_grammar(lp)
    assert fused_first_conv(lp) == 1                  # stride 1, 2x2/2 pool without padding, padded image 32x32x1


def test_cnn_strided_layers():
    lp = _plan("cnn_strided")
    assert [l.kind for l in lp.layers] == ["reshape", "conv", "conv", "pool", "conv", "reshape", "dense"]
    assert _geo(lp) == [
        ("conv", (28, 28, 1), (28, 28, 16), (3, 3), (1, 1), (1, 1, 1, 1)),
        ("conv", (28, 28, 16), (14, 14, 32), (3, 3), (2, 2), (0, 1, 0, 1)),      # pad_total = 13 * 2 + 3 - 28 = 1: bottom / right
        ("pool", (14, 14, 32), (7, 7, 32), (3, 3), (2, 2), (0, 1, 0, 1)),        # overlapping 3x3/2 windows
        ("conv", (7, 7, 32), (3, 3, 32), (3, 3), (2, 2), (0, 0, 0, 0)),          # VALID: (7 - 3) // 2 + 1
    ]
    assert lp.layers[-1].in_shape == (288,)
    assert [l.act for l in lp.layers if l.kind == "conv"] == ["Relu", "Tanh", "Relu"]
    check_grammar(lp)
    assert fused_first_conv(lp) is None               # the first conv feeds a conv, not a pool


def test_the_cnn_model_keeps_its_layers():
    lp = _plan("cnn")
    assert _geo(lp) == [
        ("conv", (28, 28, 1), (24, 24, 32), (5, 5), (1, 1), (0, 0, 0, 0)),
        ("pool", (24, 24, 32), (12, 12, 32), (2, 2), (2, 2), (0, 0, 0, 0)),
        ("conv", (12, 12, 32), (10, 10, 64), (3, 3), (1, 1), (0, 0, 0, 0)),
        ("pool", (10, 10, 64), (5, 5, 64), (2, 2), (2, 2), (0, 0, 0, 0)),
    ]


@pytest.mark.parametrize("size,k,s,padding,expect", [
    (7, 3, 2, "SAME", (4, 1, 1)),        # pad_total = 3 * 2 + 3 - 7 = 2
    (8, 3, 2, "SAME", (4, 0, 1)),        # pad_total = 1: the extra row / column goes at the bottom / right
    (28, 5, 1, "SAME", (28, 2, 2)),
    (14, 2, 2, "SAME", (7, 0, 0)),
    (13, 2, 2, "SAME", (7, 0, 1)),
    (5, 4, 1, "SAME", (5, 1, 2)),
    (7, 3, 2, "VALID", (3, 0, 0)),
    (24, 2, 2, "VALID", (12, 0, 0)),
    (3, 4, 4, "SAME", (1, 0, 1)),
])
def test_tf_padding_rule(size, k, s, padding, expect):
    assert conv_geometry(size, k, s, padding) == expect


def _compile(fn):
    return compile_graph(GraphIR.from_metagraph(build_graph(fn)), "x:0", "y:0")


def _image_net(body):
    def model():
        x = tf.placeholder(tf.float32, shape=[None, 64], name="x")
        y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
        h = body(tf.reshape(x, shape=[-1, 8, 8, 1]))
        logits = tf.layers.dense(tf.layers.flatten(h), 10)
        return tf.losses.softmax_cross_entropy(y, logits)
    return model


def test_asymmetric_same_padding_of_conv_and_pool():
    lp = _compile(_image_net(lambda img: tf.layers.max_pooling2d(tf.layers.conv2d(img, 8, 3, strides=2, padding="same"), 3, 2,
                                                                 padding="same")))
    assert _geo(lp) == [
        ("conv", (8, 8, 1), (4, 4, 8), (3, 3), (2, 2), (0, 1, 0, 1)),
        ("pool", (4, 4, 8), (2, 2, 8), (3, 3), (2, 2), (0, 1, 0, 1)),
    ]
    check_grammar(lp)
    lp = _compile(_image_net(lambda img: tf.layers.conv2d(img, 8, (3, 2), strides=(2, 1), padding="same")))
    assert _geo(lp) == [("conv", (8, 8, 1), (4, 8, 8), (3, 2), (2, 1), (0, 1, 0, 1))]
    check_grammar(lp)


def test_conv_stacks_and_conv_to_flatten_are_in_the_grammar():
    lp = _compile(_image_net(lambda img: tf.layers.conv2d(tf.layers.conv2d(img, 8, 3, padding="same"), 16, 3)))
    assert [l.kind for l in lp.layers] == ["reshape", "conv", "conv", "reshape", "dense"]
    check_grammar(lp)


def test_geometry_outside_the_plan_stays_unsupported(monkeypatch):
    def dilated(img):
        k = tf.get_variable("dilated/kernel", shape=[3, 3, 1, 8])
        return tf.nn.conv2d(img, k, [1, 1, 1, 1], "VALID", dilations=[1, 2, 2, 1])

    def pool5(img):
        return tf.layers.max_pooling2d(tf.layers.conv2d(img, 8, 3, padding="same"), 5, 1)

    def avg(img):
        return tf.layers.average_pooling2d(tf.layers.conv2d(img, 8, 3, padding="same"), 2, 2)

    def too_small(img):
        return tf.layers.conv2d(tf.layers.conv2d(img, 8, 5, strides=2), 8, 3)        # 2x2 input to a VALID 3x3 conv

    for body in (dilated, pool5, avg):
        with pytest.raises(UnsupportedGraph):
            check_grammar(_compile(_image_net(body)))
    with pytest.raises((UnsupportedGraph, ValueError)):
        check_grammar(_compile(_image_net(too_small)))
    # the K-major weight-gradient path only covers the VALID stride-1 conv + 2x2/2 pool grammar
    monkeypatch.setenv("SPARKFLOW_WGRAD_MN", "0")
    for name in ("cnn_strided", "cnn_same"):
        with pytest.raises(UnsupportedGraph):
            check_grammar(_plan(name))
    check_grammar(_plan("cnn"))
