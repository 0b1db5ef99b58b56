"""The reference's integration suite (tests/dl_runner.py:97-312 of the reference project) re-expressed against
this framework, written the way a sparkflow user would write it: through the ``sparkflow`` /
``pyspark`` / ``tensorflow`` import paths (provided by ``sparkflow_b200.compat.install()`` when the real
packages are absent).  Assertions are the reference's statistical smoke checks (errors < N of 10)."""
import os
import random
import shutil

import numpy as np
import pytest

from sparkflow_b200 import compat

compat.install()

import tensorflow as tf  # noqa: E402
from pyspark.ml.linalg import Vectors  # noqa: E402
from pyspark.ml.pipeline import Pipeline, PipelineModel  # noqa: E402
from pyspark.sql import SparkSession  # noqa: E402
from sparkflow.graph_utils import build_adam_config, build_graph, build_rmsprop_config  # noqa: E402
from sparkflow.HogwildSparkModel import HogwildSparkModel  # noqa: E402
from sparkflow.pipeline_util import PysparkPipelineWrapper  # noqa: E402
from sparkflow.tensorflow_async import SparkAsyncDL, SparkAsyncDLModel  # noqa: E402

random.seed(12345)
np.random.seed(12345)


@pytest.fixture(scope="module")
def spark():
    s = SparkSession.builder.master("local[2]").appName("sparkflow").getOrCreate()
    yield s
    s.stop()


def create_model():
    x = tf.placeholder(tf.float32, shape=[None, 2], name="x")
    layer1 = tf.layers.dense(x, 12, activation=tf.nn.relu)
    layer2 = tf.layers.dense(layer1, 7, activation=tf.nn.relu)
    out = tf.layers.dense(layer2, 1, name="outer", activation=tf.nn.sigmoid)
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    return tf.losses.mean_squared_error(y, out)


def create_random_model():
    x = tf.placeholder(tf.float32, shape=[None, 10], name="x")
    layer1 = tf.layers.dense(x, 12, activation=tf.nn.relu)
    layer2 = tf.layers.dense(layer1, 7, activation=tf.nn.relu)
    out = tf.layers.dense(layer2, 1, name="outer", activation=tf.nn.sigmoid)
    y = tf.placeholder(tf.float32, shape=[None, 1], name="y")
    return tf.losses.mean_squared_error(y, out)


def create_autoencoder():
    x = tf.placeholder(tf.float32, shape=[None, 10], name="x")
    encoder = tf.layers.dense(x, 5, activation=tf.nn.relu)
    bottle_neck = tf.layers.dense(encoder, 2, activation=tf.nn.sigmoid, name="out")
    decoder = tf.layers.dense(bottle_neck, 5, activation=tf.nn.relu)
    reconstructed = tf.layers.dense(decoder, 10)
    return tf.losses.mean_squared_error(x, reconstructed)


def calculate_errors(data):
    return sum(1 for d in data if (1 if d["predicted"] >= 0.5 else 0) != d["label"])


def gaussians(spark):
    dat = [(1.0, Vectors.dense(np.random.normal(0, 1, 10))) for _ in range(200)]
    dat += [(0.0, Vectors.dense(np.random.normal(2, 1, 10))) for _ in range(200)]
    random.shuffle(dat)
    return spark.createDataFrame(dat, ["label", "features"])


def estimator(mg, **kw):
    base = dict(inputCol="features", tensorflowGraph=mg, tfInput="x:0", tfLabel="y:0", tfOutput="outer/Sigmoid:0",
                tfOptimizer="adam", tfLearningRate=.1, iters=20, partitions=2, predictionCol="predicted", labelCol="label")
    base.update(kw)
    return SparkAsyncDL(**base)


def check(model, processed):
    data = model.transform(processed).take(10)
    assert calculate_errors(data) < len(data)


def test_save_model(spark, tmp_path):
    processed = gaussians(spark)
    fitted = estimator(build_graph(create_random_model)).fit(processed)
    path = str(tmp_path / "saved_model")
    fitted.save(path)
    check(SparkAsyncDLModel.load(path), processed)


def test_save_pipeline(spark, tmp_path):
    processed = gaussians(spark)
    p = Pipeline(stages=[estimator(build_graph(create_random_model))]).fit(processed)
    path = str(tmp_path / "example_pipeline")
    p.write().overwrite().save(path)
    p.write().overwrite().save(path)          # overwrite really overwrites
    loaded = PysparkPipelineWrapper.unwrap(PipelineModel.load(path))
    assert isinstance(loaded.stages[0], SparkAsyncDLModel)
    check(loaded, processed)


def test_adam_optimizer_options(spark, capsys):
    processed = gaussians(spark)
    options = build_adam_config(learning_rate=0.1, beta1=0.85, beta2=0.98, epsilon=1e-8)
    model = estimator(build_graph(create_random_model), iters=25, verbose=1, optimizerOptions=options).fit(processed)
    check(model, processed)
    out = capsys.readouterr().out
    assert "Partition Id:" in out and "Iteration: 24, Loss:" in out      # reference log format


def test_small_sparse(spark):
    xor = [(0.0, Vectors.sparse(2, [0, 1], [0.0, 0.0])), (0.0, Vectors.sparse(2, [0, 1], [1.0, 1.0])),
           (1.0, Vectors.sparse(2, [0], [1.0])), (1.0, Vectors.sparse(2, [1], [1.0]))]
    processed = spark.createDataFrame(xor, ["label", "features"])
    model = estimator(build_graph(create_model), iters=35).fit(processed)
    assert model.transform(processed).collect() is not None


def test_spark_hogwild(spark):
    xor = [(0.0, Vectors.dense(np.array([0.0, 0.0]))), (0.0, Vectors.dense(np.array([1.0, 1.0]))),
           (1.0, Vectors.dense(np.array([1.0, 0.0]))), (1.0, Vectors.dense(np.array([0.0, 1.0])))]
    processed = spark.createDataFrame(xor, ["label", "features"]).coalesce(1).rdd.map(lambda x: (np.asarray(x["features"]), x["label"]))
    first_graph = tf.Graph()
    with first_graph.as_default():
        create_model()
        mg = compat.json_format.MessageToJson(tf.train.export_meta_graph())
    spark_model = HogwildSparkModel(tensorflowGraph=mg, iters=10, tfInput="x:0", tfLabel="y:0",
                                    optimizer=tf.train.AdamOptimizer(learning_rate=.1), master_url="localhost:5000")
    try:
        weights = spark_model.train(processed)
        assert len(weights) == 6 and weights[0].shape == (2, 12)
    except Exception:
        spark_model.stop_server()
        raise


def test_overlapping_guassians(spark):
    processed = gaussians(spark)
    check(estimator(build_graph(create_random_model), iters=35).fit(processed), processed)


def test_rmsprop(spark):
    processed = gaussians(spark)
    options = build_rmsprop_config(learning_rate=0.1, decay=0.95, momentum=0.1, centered=False)
    check(estimator(build_graph(create_random_model), tfOptimizer="rmsprop", iters=25, optimizerOptions=options).fit(processed), processed)


def test_multi_partition_shuffle(spark):
    processed = gaussians(spark)
    check(estimator(build_graph(create_random_model), partitionShuffles=2).fit(processed), processed)


def test_auto_encoder(spark):
    processed = gaussians(spark)
    model = SparkAsyncDL(inputCol="features", tensorflowGraph=build_graph(create_autoencoder), tfInput="x:0", tfLabel=None,
                         tfOutput="out/Sigmoid:0", tfOptimizer="adam", tfLearningRate=.001, iters=10, predictionCol="predicted",
                         partitions=4, miniBatchSize=10, verbose=1).fit(processed)
    encoded = model.transform(processed).take(10)
    assert len(encoded[0]["predicted"]) == 2


def test_change_port(spark):
    processed = gaussians(spark)
    check(estimator(build_graph(create_random_model), iters=35, port=3000).fit(processed), processed)


# ---- modes the reference never tested (SURVEY.md section 4) ----------------------------------------
def test_acquire_lock_mode(spark):
    processed = gaussians(spark)
    check(estimator(build_graph(create_random_model), iters=25, acquireLock=True).fit(processed), processed)


def test_mini_stochastic_iters_mode_a(spark):
    processed = gaussians(spark)
    check(estimator(build_graph(create_random_model), iters=60, miniBatchSize=50, miniStochasticIters=3).fit(processed), processed)


def test_full_batch_mode_c(spark):
    processed = gaussians(spark)
    check(estimator(build_graph(create_random_model), iters=120, miniBatchSize=-1).fit(processed), processed)


def test_loss_callback_and_counters(spark):
    processed = gaussians(spark)
    rdd = processed.rdd.map(lambda r: (np.asarray(r["features"]), r["label"])).coalesce(2)
    seen = []
    m = HogwildSparkModel(tensorflowGraph=build_graph(create_random_model), iters=4, tfInput="x:0", tfLabel="y:0",
                          optimizer=tf.train.AdamOptimizer(0.05), mini_batch=100, loss_callback=lambda l, i, pid: seen.append((l, i, pid)))
    m.train(rdd)
    assert len(seen) == 8 and {i for _, i, _ in seen} == {0, 1, 2, 3} and len({pid for _, _, pid in seen}) == 2
    assert all(np.isfinite(l) for l, _, _ in seen)


def test_handle_model_foreach_partition_and_module_helpers(spark):
    """the reference's own driver loop, spelled out: ``rdd.foreachPartition(handle_model)`` against a running server,
    then ``get_server_weights`` / ``put_deltas_to_server`` by master url (HogwildSparkModel.py:22-100, 246-272)"""
    from sparkflow.HogwildSparkModel import get_server_weights, handle_model, put_deltas_to_server

    rdd = gaussians(spark).rdd.map(lambda r: (np.asarray(r["features"]), r["label"])).coalesce(2)
    mg = build_graph(create_random_model)
    m = HogwildSparkModel(tensorflowGraph=mg, iters=3, tfInput="x:0", tfLabel="y:0", optimizer=tf.train.AdamOptimizer(0.05),
                          master_url="localhost:5011", port=5011, engine="torch", seed=3)
    try:
        w0 = get_server_weights("localhost:5011")
        seen = []
        rdd.foreachPartition(lambda part: handle_model(part, mg, "x:0", tfLabel="y:0", master_url="localhost:5011", iters=3,
                                                       mini_batch_size=50, loss_callback=lambda l, i, pid: seen.append((i, pid))))
        w1 = get_server_weights("localhost:5011")
        assert len(seen) == 6 and len({pid for _, pid in seen}) == 2
        assert any(not np.allclose(a, b) for a, b in zip(w0, w1))
        # one explicit delta = one optimizer step on the master
        put_deltas_to_server([np.ones_like(w) for w in w1], "localhost:5011")
        w2 = get_server_weights("localhost:5011")
        assert all(np.all(b < a) for a, b in zip(w1, w2))          # adam step against an all-ones gradient lowers every weight
        with pytest.raises(ValueError):
            handle_model(iter([]), mg + " ", "x:0", tfLabel="y:0", master_url="localhost:5011")
        m.start_service(mg, None, 5011)                              # the reference's service entry point: idempotent here
    finally:
        m.stop_server()
    with pytest.raises(ConnectionError):
        get_server_weights("localhost:5011")
