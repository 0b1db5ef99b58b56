"""End-to-end numerics of the compiled H100 step (pull -> fwd -> loss -> bwd -> push) against the
PyTorch-autograd oracle running the reference semantics on the CPU."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import compile_graph
from sparkflow_b200.ops.layout import ParamLayout
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs
from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer
from sparkflow_b200.parallel.worker import B200Engine, TorchEngine

CASES = {
    "cnn": ("x:0", "y:0", 784, 10, "onehot"),
    "simple_dnn": ("x:0", "y:0", 784, 10, "onehot"),
    "autoencoder": ("x:0", None, 784, 0, None),
    "test_mlp": ("x:0", "y:0", 10, 1, "binary"),
    "test_autoencoder": ("x:0", None, 10, 0, None),
}


def _data(n, d, c, kind, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.random((n, d), dtype=np.float32)
    if kind == "onehot":
        Y = np.eye(c, dtype=np.float32)[rng.integers(0, c, n)]
    elif kind == "binary":
        Y = rng.integers(0, 2, (n, 1)).astype(np.float32)
    else:
        Y = None
    return X, Y


def _setup(name, spec, lock=False, pull_mode="copy", served=False, dbuf=False):
    tf_in, tf_lab, d, c, kind = CASES[name]
    ir = GraphIR.from_metagraph(zoo.build(name))
    lp = compile_graph(ir, tf_in, tf_lab)
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    dev = torch.device("cuda:0")
    master = MasterState(lay, spec, dev, n_mailboxes=1 if served else 0)
    w0 = GraphProgram(ir).init_weights(seed=1)
    master.load_weights(w0)
    if served:
        master.start_applier(lock, scope_sys=False, grid=32, dbuf=dbuf)
    worker = DeviceWorker(ir, tf_in, tf_lab, spec, master, acquire_lock=lock, pull_mode=pull_mode, shared=False)
    return ir, master, worker, w0, (tf_in, tf_lab, d, c, kind)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("lock", [False, True])
def test_compiled_step_tracks_oracle(name, lock):
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    ir, master, worker, w0, (tf_in, tf_lab, d, c, kind) = _setup(name, spec, lock)
    X, Y = _data(256, d, c, kind)
    eng = B200Engine(worker)
    eng.load_partition(X, Y)
    ps = ParameterServer(w0, spec, acquire_lock=lock)
    ref = TorchEngine(ir, tf_in, tf_lab, LocalTransport(ps))
    ref.load_partition(X, Y)
    rows = [slice(0, 64), slice(64, 128), np.arange(100, 164), slice(192, 256), slice(0, 64)]
    for r in rows:
        eng.train(r, pull=True)
        ref.train(r, pull=True)
    eng.finish()
    got, exp = master.weights(), ps.weights()
    for a, b, v in zip(got, exp, ir.trainable):
        # adam steps are +-lr per element; bf16 forward/backward may flip the sign of tiny gradients
        assert np.abs(a - b).max() < 5 * 0.001 * len(rows), v.name
        assert np.mean(np.abs(a - b)) < 0.35 * 0.001 * len(rows), v.name
    cnt = master.counters()
    assert cnt["pushes"] == len(rows) and cnt["lock"] == 0
    # loss of the last step agrees with the oracle's loss on the same batch before its update
    loss_gpu = worker.partition_loss(eng.X, eng.Y)
    loss_ref = GraphProgram(ir).loss(ref._feed(slice(0, 256)), got)
    assert abs(loss_gpu - loss_ref) < 2e-2 * max(1.0, abs(loss_ref))
    master.close()


def test_training_reduces_loss_and_predicts():
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.002))
    ir, master, worker, w0, (tf_in, tf_lab, d, c, kind) = _setup("simple_dnn", spec)
    rng = np.random.default_rng(3)
    centers = rng.normal(0, 1, (10, 784)).astype(np.float32)
    lab = rng.integers(0, 10, 3000)
    X = centers[lab] + 0.3 * rng.normal(0, 1, (3000, 784)).astype(np.float32)
    Y = np.eye(10, dtype=np.float32)[lab]
    eng = B200Engine(worker)
    eng.load_partition(X, Y)
    l0 = eng.partition_loss()
    for it in range(30):
        for r in range(0, 3000, 300):
            eng.train(slice(r, r + 300), pull=True)
    eng.finish()
    l1 = eng.partition_loss()
    assert l1 < 0.2 * l0, (l0, l1)
    # prediction through the forward-only plan (+ArgMax kernel)
    pred = worker.predict(X[:500], upto=2, post="ArgMax")
    assert (pred.astype(np.int64) == lab[:500]).mean() > 0.95
    master.close()


@pytest.mark.parametrize("pull_mode", ["copy", "direct"])
def test_graph_replay_equals_eager(pull_mode):
    spec = OptimizerSpec.from_tf_kwargs("gradient_descent", dict(learning_rate=0.05))
    outs = []
    for use_graphs in (False, True):
        ir, master, worker, w0, (tf_in, tf_lab, d, c, kind) = _setup("test_mlp", spec, pull_mode=pull_mode)
        worker.use_graphs = use_graphs
        X, Y = _data(128, d, c, kind, seed=5)
        eng = B200Engine(worker)
        eng.load_partition(X, Y)
        for _ in range(6):
            eng.train(slice(0, 128), pull=True)
        eng.finish()
        outs.append(master.weights())
        master.close()
    for a, b in zip(*outs):
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("lock,dbuf", [(False, False), (True, False), (True, True)])
def test_served_push_mailbox_applier_tracks_oracle(lock, dbuf):
    """push = post to the mailbox + applier kernels on the master GPU; same numbers as direct mode.  dbuf: lock mode
    with the double-buffered publish (pulls register with one atomic and copy the complete buffer, no RW lock)."""
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    ir, master, worker, w0, (tf_in, tf_lab, d, c, kind) = _setup("simple_dnn", spec, lock, served=True, dbuf=dbuf)
    assert worker.served and master.applier.alive() and worker.use_dbuf == dbuf and master.dbuf_active == dbuf
    X, Y = _data(256, d, c, kind)
    eng = B200Engine(worker)
    eng.load_partition(X, Y)
    ps = ParameterServer(w0, spec, acquire_lock=lock)
    ref = TorchEngine(ir, tf_in, tf_lab, LocalTransport(ps))
    ref.load_partition(X, Y)
    rows = [slice(0, 64), slice(64, 128), slice(128, 192), slice(192, 256)] * 3
    for r in rows:
        eng.train(r, pull=True)          # each pull waits until the applier has consumed this worker's previous post
        ref.train(r, pull=True)
    eng.finish()
    import time
    t0 = time.time()
    while master.counters()["pushes"] < len(rows) and time.time() - t0 < 10:
        time.sleep(0.01)
    cnt = master.counters()
    assert cnt["pushes"] == len(rows) and cnt["lock"] == 0, cnt
    for a, b, v in zip(master.weights(), ps.weights(), ir.trainable):
        assert np.abs(a - b).max() < 5 * 0.001 * len(rows), v.name
        assert np.mean(np.abs(a - b)) < 0.35 * 0.001 * len(rows), v.name
    assert master.applier.alive()
    if dbuf:
        # stopping the applier settles the publish on buffer 0: it must equal the bf16 image of the final parameters
        master.stop_applier()
        lay = master.layout
        pub = lay.publish_reference(lay.flatten(master.weights()))
        np.testing.assert_allclose(master.shadow.float().cpu().numpy(), torch.from_numpy(pub).to(torch.bfloat16).float().numpy(), rtol=0, atol=1e-2)
        flat = lay.flatten(master.weights())
        np.testing.assert_array_equal(master.vec_pub[0][:lay.vec_count].cpu().numpy(), flat[lay.vec_offset:lay.vec_offset + lay.vec_count])
        assert master.counters()["lock"] == 0 and int(master.ctrl[master.C.CTRL_PUB].item()) == 0
    master.close()
    assert master.applier is None


@pytest.mark.parametrize("opt", ["adam", "momentum", "rmsprop"])
@pytest.mark.parametrize("max_batch", [1, 3, 8])
def test_applier_batch_is_sequential_pushes(opt, max_batch):
    """Four gradients posted at once are applied in ONE pass over the state (or max_batch at a time), and the result
    equals four separate optimizer steps in mailbox order, each with its own step number - no gradient aggregation."""
    import time
    kw = dict(learning_rate=0.01)
    if opt == "momentum":
        kw["momentum"] = 0.9
    spec = OptimizerSpec.from_tf_kwargs(opt, kw)
    ir = GraphIR.from_metagraph(zoo.build("test_mlp"))
    lp = compile_graph(ir, "x:0", "y:0")
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    dev = torch.device("cuda:0")
    n_w = 4
    master = MasterState(lay, spec, dev, n_mailboxes=n_w)
    w0 = GraphProgram(ir).init_weights(seed=3)
    master.load_weights(w0)
    rng = np.random.default_rng(5)
    grads = [[rng.standard_normal(s).astype(np.float32) for _, s in ir.param_shapes()] for _ in range(n_w)]
    ps = ParameterServer(w0, spec, acquire_lock=True)
    boxes = master._bytes[master.ml.mailboxes:master.ml.mailboxes + n_w * master.ml.mailbox_stride * 4].view(torch.float32)
    boxes = boxes.view(n_w, master.ml.mailbox_stride)
    flags = master._bytes[master.ml.flags:master.ml.flags + n_w * master.C.MB_WORDS * 4].view(torch.int32).view(n_w, master.C.MB_WORDS)
    flags.zero_()
    for w in range(n_w):
        boxes[w, :lay.total] = torch.from_numpy(lay.flatten(grads[w])).to(dev)
        LocalTransport(ps).push(grads[w])
    flags[:, 0] = 1                                    # POSTED = 1 for every worker before the applier starts
    torch.cuda.current_stream(dev).synchronize()
    master.start_applier(True, scope_sys=False, grid=8, max_batch=max_batch)
    t0 = time.time()
    while master.counters()["pushes"] < n_w and time.time() - t0 < 10:
        time.sleep(0.01)
    cnt = master.counters()
    assert cnt["pushes"] == n_w and cnt["step"] == n_w and cnt["version"] == n_w and cnt["lock"] == 0, cnt
    assert flags[:, master.C.MB_APPLIED].cpu().tolist() == [1] * n_w
    for a, b, v in zip(master.weights(), ps.weights(), ir.trainable):
        np.testing.assert_allclose(a, b, rtol=2e-5, atol=2e-6, err_msg=v.name)
    # published bf16 operands match the final fp32 parameters
    pub = lay.publish_reference(lay.flatten(master.weights()))
    np.testing.assert_allclose(master.shadow.float().cpu().numpy(), torch.from_numpy(pub).to(torch.bfloat16).float().numpy(), rtol=0, atol=1e-2)
    master.close()


@pytest.mark.parametrize("partition", ["pinned", "resident"])
@pytest.mark.parametrize("served", [False, True])
def test_train_contiguous_native_loop_tracks_oracle(partition, served, monkeypatch):
    """the C++ StepDriver loop walks the same minibatches as the oracle, before and after a shuffle of the partition:
    a pinned one (copy-engine H2D per step, physical shuffle) and an HBM-resident one (device-side gather / shuffle)"""
    monkeypatch.setenv("SPARKFLOW_PARTITION", partition)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    ir, master, worker, w0, (tf_in, tf_lab, d, c, kind) = _setup("simple_dnn", spec, True, served=served, dbuf=served)
    X, Y = _data(640, d, c, kind)
    eng = B200Engine(worker)
    assert eng.partition_mode == partition
    eng.load_partition(X, Y)
    ps = ParameterServer(w0, spec, acquire_lock=True)
    ref = TorchEngine(ir, tf_in, tf_lab, LocalTransport(ps))
    ref.load_partition(X, Y)
    starts = [0, 64, 128, 192, 256, 320, 384, 448, 512, 576, 0]
    eng.train_contiguous(starts, 64, pull=True)
    for s0 in starts:
        ref.train(slice(s0, s0 + 64), pull=True)
    eng.finish()
    # loss of the LAST minibatch (rows 0..63) evaluated with the weights that step pulled
    l_dev = eng.last_loss()
    l_ref = float(ref.prog.loss(ref._feed(slice(0, 64)), ref.weights))
    assert abs(l_dev - l_ref) < 0.05 * max(1.0, abs(l_ref)), (l_dev, l_ref)
    order = np.random.default_rng(3).permutation(640)
    eng.permute(order)
    ref.load_partition(X[order], Y[order])
    eng.train_contiguous(starts[:5], 64, pull=True)
    for s0 in starts[:5]:
        ref.train(slice(s0, s0 + 64), pull=True)
    # explicit row ids (the reference's mini_stochastic_iters mode) index the shuffled partition
    picks = [np.random.default_rng(10 + i).choice(640, 64, replace=False) for i in range(2)]
    for rows in picks:
        eng.train(rows, pull=True)
        ref.train(rows, pull=True)
    eng.train_contiguous([256], 64, pull=True)
    ref.train(slice(256, 320), pull=True)
    eng.finish()
    import time
    n = len(starts) + 5 + 3
    t0 = time.time()
    while master.counters()["pushes"] < n and time.time() - t0 < 10:
        time.sleep(0.01)
    assert master.counters()["pushes"] == n
    for a, b, v in zip(master.weights(), ps.weights(), ir.trainable):
        assert np.abs(a - b).max() < 5 * 0.001 * n, v.name
        assert np.mean(np.abs(a - b)) < 0.35 * 0.001 * n, v.name
    l_ref = float(ref.prog.loss(ref._feed(slice(256, 320)), ref.weights))
    assert abs(eng.last_loss() - l_ref) < 0.05 * max(1.0, abs(l_ref)), (eng.last_loss(), l_ref)
    master.close()


def test_fused_dropout_mask_statistics_and_gradients():
    """K13: tf.nn.dropout after a dense layer runs inside the compiled plan (Philox mask in the GEMM epilogue).  The mask
    is recovered from the stored activation; forward statistics and every gradient are checked against PyTorch given
    that observed mask (reference semantics: keep with prob p, scale by 1/p - tf.nn.dropout; ml_util.py:70-71)."""
    from sparkflow_b200.graph import tfcompat as tf
    from sparkflow_b200.graph_utils import build_graph

    def model():
        x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
        y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
        kp = tf.placeholder_with_default(0.5, shape=[], name="keep_prob")
        h1 = tf.nn.dropout(tf.layers.dense(x, 256, activation=tf.nn.relu), keep_prob=kp)
        h2 = tf.layers.dense(h1, 128, activation=tf.nn.tanh)
        h2 = tf.layers.dropout(h2, rate=0.25, training=True)
        logits = tf.layers.dense(h2, 10)
        tf.argmax(logits, 1, name="out")
        return tf.losses.softmax_cross_entropy(y, logits)

    spec = OptimizerSpec.from_tf_kwargs("gradient_descent", dict(learning_rate=0.0))
    ir = GraphIR.from_metagraph(build_graph(model))
    lp = compile_graph(ir, "x:0", "y:0")
    assert [round(l.dropout_keep, 2) for l in lp.layers] == [0.5, 0.75, 0.0]
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    dev = torch.device("cuda:0")
    master = MasterState(lay, spec, dev)
    w0 = GraphProgram(ir).init_weights(seed=2)
    w0 = [w if w.ndim > 1 else (0.1 * np.random.default_rng(1).standard_normal(w.shape)).astype(np.float32) for w in w0]
    master.load_weights(w0)
    worker = DeviceWorker(ir, "x:0", "y:0", spec, master, shared=False, use_graphs=False)
    B = 256
    X, Y = _data(B, 784, 10, "onehot", seed=5)
    plan, bufs = worker.build_plan(B, 0, with_pull=True, with_push=False)
    with torch.cuda.stream(worker.stream):
        bufs.x_stage.copy_(torch.from_numpy(X))
        bufs.y_stage.copy_(torch.from_numpy(Y))
        plan.run(worker.stream.cuda_stream)
    worker.stream.synchronize()
    dbg = worker.last_debug
    dense = [i for i, l in enumerate(lp.layers) if l.kind == "dense"]
    a1 = dbg[dense[1]]["a_in"].float()[:, :256].cpu()          # dropout(relu(x W0 + b0), keep 0.5) as consumed by layer 1
    a2 = dbg[dense[2]]["a_in"].float()[:, :128].cpu()          # dropout(tanh(.), keep 0.75)
    xb = torch.from_numpy(X).to(torch.bfloat16).float()
    W = [torch.from_numpy(w).to(torch.bfloat16).float() if w.ndim > 1 else torch.from_numpy(w) for w in w0]
    h1 = torch.relu(xb @ W[0] + W[1])
    m1 = (a1 != 0).float()
    pos = h1 > 1e-3
    kept = (m1[pos]).mean().item()
    assert 0.47 < kept < 0.53, kept                              # keep probability 0.5
    assert torch.allclose(a1[pos & (m1 > 0)], 2.0 * h1[pos & (m1 > 0)], rtol=3e-2, atol=3e-2)   # survivors scaled by 1/keep
    h2 = torch.tanh(a1 @ W[2] + W[3])
    m2 = (a2 != 0).float()
    big = h2.abs() > 1e-2
    assert 0.72 < m2[big].mean().item() < 0.78
    assert torch.allclose(a2[big & (m2 > 0)], h2[big & (m2 > 0)] / 0.75, rtol=3e-2, atol=3e-2)
    # the two layers' masks are different streams, rows differ, columns differ
    assert (m1[0] != m1[1]).any() and (m1[:, 0] != m1[:, 1]).any()
    # ---- gradients given the observed masks (autograd on the same computation) ----
    Wt = [w.clone().requires_grad_(True) for w in W]
    xh = xb
    z1 = torch.relu(xh @ Wt[0] + Wt[1]) * m1 * 2.0
    z2 = torch.tanh(z1.to(torch.bfloat16).float() @ Wt[2] + Wt[3]) * m2 / 0.75
    logits = z2.to(torch.bfloat16).float() @ Wt[4] + Wt[5]
    loss = -(torch.from_numpy(Y) * torch.log_softmax(logits, 1)).sum(1).mean()
    loss.backward()
    got = lay.unflatten(worker.grads.cpu().numpy())
    for g, w, v in zip(got, Wt, ir.trainable):
        ref = w.grad.numpy()
        scale = max(np.abs(ref).max(), 1e-6)
        assert np.abs(g - ref).max() < 6e-2 * scale, (v.name, np.abs(g - ref).max(), scale)
    assert abs(float(worker.loss_acc.cpu()[0]) - float(loss)) < 2e-2 * max(1.0, float(loss))
    # a second step draws a different mask only when the step counter moves: without a push the counter is unchanged
    master.close()
