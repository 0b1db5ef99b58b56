"""MNIST multi-layer perceptron (784-256-256-10) through the Spark-ML pipeline API: VectorAssembler + OneHotEncoder +
SparkAsyncDL, saved, re-loaded through the carrier format and scored.  Same workload as the reference's simple_dnn
example; here every partition trains on an H100 (or a CPU thread) against the device-resident parameter server.

    python examples/simple_dnn.py [--rows N] [--iters K]           one worker per GPU / thread in this process
    torchrun --nproc-per-node 8 examples/simple_dnn.py             one rank per H100, master on rank 0's GPU
"""
from _common import Stopwatch, mnist_frame, parse_args, pixel_columns

import tensorflow as tf
from pyspark.ml.evaluation import MulticlassClassificationEvaluator
from pyspark.ml.feature import OneHotEncoder, VectorAssembler
from pyspark.ml.pipeline import Pipeline, PipelineModel
from sparkflow.graph_utils import build_adam_config, build_graph
from sparkflow.pipeline_util import PysparkPipelineWrapper
from sparkflow.tensorflow_async import SparkAsyncDL

HIDDEN = (256, 256)
CLASSES = 10
BATCH = 300


def mlp():
    """Graph function for build_graph: placeholders x / y, ReLU hidden layers, an ArgMax node named `out`, softmax-CE loss."""
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, CLASSES], name="y")
    h = x
    for width in HIDDEN:
        h = tf.layers.dense(h, width, activation=tf.nn.relu, kernel_initializer=tf.glorot_uniform_initializer())
    logits = tf.layers.dense(h, CLASSES, kernel_initializer=tf.glorot_uniform_initializer())
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def main():
    args = parse_args(__doc__.splitlines()[0], iters=50)
    spark, frame = mnist_frame(args)
    stages = [
        VectorAssembler(inputCols=pixel_columns(frame), outputCol="features"),
        OneHotEncoder(inputCol="_c0", outputCol="labels", dropLast=False),
        SparkAsyncDL(inputCol="features", labelCol="labels", predictionCol="predicted", tensorflowGraph=build_graph(mlp),
                     tfInput="x:0", tfLabel="y:0", tfOutput="out:0", tfOptimizer="adam",
                     optimizerOptions=build_adam_config(learning_rate=0.001, beta1=0.9, beta2=0.999),
                     miniBatchSize=BATCH, miniStochasticIters=1, shufflePerIter=True, iters=args.iters,
                     partitions=args.partitions, verbose=0 if args.quiet else 1),
    ]
    with Stopwatch("simple_dnn", frame.count(), args.iters, BATCH):
        fitted = Pipeline(stages=stages).fit(frame)
    target = args.out or "/tmp/simple_dnn"
    fitted.write().overwrite().save(target)
    restored = PysparkPipelineWrapper.unwrap(PipelineModel.load(target))
    accuracy = MulticlassClassificationEvaluator(labelCol="_c0", predictionCol="predicted", metricName="accuracy").evaluate(
        restored.transform(frame))
    print("Test Error = %g" % (1.0 - accuracy))
    spark.stop()


if __name__ == "__main__":
    main()
