"""MNIST convolutional network (conv 5x5x32 - pool - conv 3x3x64 - pool - dense 10) trained with SparkAsyncDL.
On an H100 the step is the compiled sm_90a plan: im2col + wgmma GEMMs, pooling with an arg-max mask, pooling backward
fused with the ReLU gradient.  Same workload as the reference's cnn example.

    python examples/cnn_example.py [--rows N] [--iters K]
"""
from _common import Stopwatch, mnist_frame, parse_args, pixel_columns

import tensorflow as tf
from pyspark.ml.feature import OneHotEncoder, VectorAssembler
from pyspark.ml.pipeline import Pipeline
from sparkflow.graph_utils import build_graph
from sparkflow.tensorflow_async import SparkAsyncDL

CONVS = ((32, 5), (64, 3))        # (filters, kernel size); each followed by 2x2 max pooling
BATCH = 300


def convnet():
    flat = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    onehot = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    feature_map = tf.reshape(flat, shape=[-1, 28, 28, 1])
    for filters, ksize in CONVS:
        feature_map = tf.layers.conv2d(feature_map, filters, ksize, activation=tf.nn.relu)
        feature_map = tf.layers.max_pooling2d(feature_map, 2, 2)
    logits = tf.layers.dense(tf.layers.flatten(feature_map), 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(onehot, logits)


def main():
    args = parse_args(__doc__.splitlines()[0], iters=50)
    spark, frame = mnist_frame(args, driver_memory="4g")
    trainer = SparkAsyncDL(inputCol="features", labelCol="labels", predictionCol="predicted", tensorflowGraph=build_graph(convnet),
                           tfInput="x:0", tfLabel="y:0", tfOutput="out:0", tfOptimizer="adam", tfLearningRate=1e-4,
                           miniBatchSize=BATCH, miniStochasticIters=-1, shufflePerIter=True, iters=args.iters,
                           partitions=args.partitions, verbose=0 if args.quiet else 1)
    pipeline = Pipeline(stages=[VectorAssembler(inputCols=pixel_columns(frame), outputCol="features"),
                                OneHotEncoder(inputCol="_c0", outputCol="labels", dropLast=False), trainer])
    with Stopwatch("cnn", frame.count(), args.iters, BATCH):
        fitted = pipeline.fit(frame)
    target = args.out or "/tmp/cnn"
    fitted.write().overwrite().save(target)
    first = fitted.transform(frame).take(1)[0]
    print(f"saved {target}; label {first['_c0']} -> predicted {first['predicted']}")
    spark.stop()


if __name__ == "__main__":
    main()
