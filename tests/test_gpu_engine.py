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
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout
from sparkflow_b200.ops.optimizers import OptimizerSpec, apply_update
from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs
from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer
from sparkflow_b200.parallel.worker import B200Engine, TorchEngine
from push_helpers import OPTIMIZERS, wait_pushes

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


def _applier_gradients(lay, n, rng):
    """``n`` flat gradients whose magnitudes span 1e-4 .. 10 (either side of every l1 threshold of OPTIMIZERS), about a
    tenth of them exact zeros, and a ``quiet`` set of elements that start at 0 and never see a gradient above 1e-6: the
    l1-regularised rules (FTRL, proximal, AdagradDA) clamp those to 0 by a margin of 100x or more."""
    valid = lay.valid_mask()
    quiet = valid & (rng.random(lay.total) < 0.25)
    grads = []
    for _ in range(n):
        g = np.sign(rng.standard_normal(lay.total)) * 10.0 ** rng.uniform(-4, 1, lay.total)
        g[quiet] = 1e-6 * rng.uniform(-1, 1, int(quiet.sum()))
        g[rng.random(lay.total) < 0.1] = 0.0
        g[~valid] = 0.0
        grads.append(g.astype(np.float32))
    return grads, quiet


def _within(what, got, ref, atol, rtol=2e-5):
    """(max |got - ref|, worst |got - ref| / (atol + rtol |ref|)); fails when that ratio exceeds 1"""
    err = np.abs(got - ref)
    ratio = err / (atol + rtol * np.abs(ref))
    assert (ratio <= 1).all(), f"{what}: {int((ratio > 1).sum())} elements off, worst at {ratio.max():.2f}x the tolerance"
    return float(err.max(initial=0.0)), float(ratio.max(initial=0.0))


# every optimizer with all posts of a pass batched (max_batch 8), and the step-number dependent rules (Adam's bias
# correction, AdagradDA's l1 * t / l2 * t) also one and three pushes per pass
APPLIER_CASES = [pytest.param(mb, opt, kw, model, kind, id=f"{mb}-{opt}-kw{i}-{model}-{kind}")
                 for i, (opt, kw) in enumerate(OPTIMIZERS) for mb in ((1, 3, 8) if opt in ("adam", "adagrad_da") else (8,))
                 for model in ("test_mlp", "simple_dnn") for kind in ("served", "sharded")]


@pytest.mark.parametrize("max_batch,opt,kw,model,master_kind", APPLIER_CASES)
def test_applier_batch_is_sequential_pushes(max_batch, opt, kw, model, master_kind):
    """Four posted gradients are applied max_batch at a time, in ONE pass over the state per batch, and the result equals
    four separate optimizer steps in application order (round-robin from the cursor), the k-th gradient of a pass with
    step number t0 + k - no gradient aggregation.  Every optimizer, against ``apply_update`` in float64 (parameters and
    every slot), on test_mlp (scalar tiles, fewer tiles than CTAs) and simple_dnn (several tiles per CTA: the pipelined
    tile loop).  served: one master with four mailboxes; sharded: two shards (two workers, so two rounds of two posts),
    whose appliers hand the mailboxes back zeroed (mb_zero)."""
    spec = OptimizerSpec.from_tf_kwargs(opt, kw)
    ir = GraphIR.from_metagraph(zoo.build(model))
    lp = compile_graph(ir, "x:0", "y:0")
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    dev = torch.device("cuda:0")
    C = native.cuda_ext()
    n_g = 4
    rng = np.random.default_rng(5)
    w0 = [(0.1 * rng.standard_normal(s)).astype(np.float32) for _, s in ir.param_shapes()]
    grads, quiet = _applier_gradients(lay, n_g, rng)
    flat0 = lay.flatten(w0)
    flat0[quiet] = 0.0
    w0 = lay.unflatten(flat0)
    valid = lay.valid_mask()
    n_tiles = int(lay.tile_map().shape[0])
    if master_kind == "served":
        master = MasterState(lay, spec, dev, n_mailboxes=n_g)
        master.load_weights(w0)
        boxes = master._bytes[master.ml.mailboxes:master.ml.mailboxes + n_g * master.ml.mailbox_stride * 4].view(torch.float32)
        boxes = boxes.view(n_g, master.ml.mailbox_stride)
        flags = master._bytes[master.ml.flags:master.ml.flags + n_g * C.MB_WORDS * 4].view(torch.int32).view(n_g, C.MB_WORDS)
        flags.zero_()
        for w in range(n_g):
            boxes[w, :lay.total] = torch.from_numpy(grads[w]).to(dev)
        flags[:, 0] = 1                                    # POSTED = 1 for every worker before the applier starts
        torch.cuda.current_stream(dev).synchronize()
        grid = 8
        master.start_applier(True, scope_sys=False, grid=grid, max_batch=max_batch)
        tiles_per_cta = [n_tiles / grid]
        wait_pushes(master, n_g)
        cnt = master.counters()
        assert cnt["pushes"] == n_g and cnt["step"] == n_g and cnt["version"] == n_g and cnt["lock"] == 0, cnt
        assert flags[:, C.MB_APPLIED].cpu().tolist() == [1] * n_g
    else:
        from sparkflow_b200.parallel.device_engine import _view
        from sparkflow_b200.parallel.dist import DistContext
        from sparkflow_b200.parallel.sharded import ShardedMaster

        master = ShardedMaster(lay, spec, DistContext(), [dev, dev], mb_zero=True)
        master.load_weights(w0)
        n_w = master.n
        owned = master._owners()
        tiles_per_cta = [(master.bounds[s + 1] - master.bounds[s]) / master.applier_grid(s) for s in range(n_w)]

        def flags(s, w):
            return _view(master.posted_ptr(s, w), C.MB_WORDS * 4, torch.int32, dev)

        def box(s, w):
            return _view(master.mailbox_ptr(s, w), lay.total * 4, torch.float32, dev)

        for rnd in range(n_g // n_w):
            # each shard's mailbox receives only the elements it owns, as the routed wgrad epilogues store them
            for s in range(n_w):
                idx = owned[s].to(dev)
                for w in range(n_w):
                    box(s, w).index_copy_(0, idx, torch.from_numpy(grads[rnd * n_w + w]).to(dev).index_select(0, idx))
                    flags(s, w)[0] = rnd + 1
            torch.cuda.current_stream(dev).synchronize()
            master.start_applier(False, max_batch=max_batch)
            wait_pushes(master, (rnd + 1) * n_w)
            master.stop_applier()
            cnt = master.counters()
            assert cnt["pushes"] == (rnd + 1) * n_w and cnt["step"] == (rnd + 1) * n_w, cnt
            assert all(int(flags(s, w)[C.MB_APPLIED]) == rnd + 1 for s in range(n_w) for w in range(n_w))
            for s in range(n_w):
                for w in range(n_w):
                    assert not bool(box(s, w).any()), f"shard {s} did not hand mailbox {w} back zeroed (mb_zero)"
    # the pipelined tile loop runs where a CTA owns more than one tile
    assert all(t > 1 for t in tiles_per_cta) == (model == "simple_dnn"), tiles_per_cta
    # float64 reference (on the device: 269k elements): the four gradients in application order, step numbers 1..4
    p_ref = torch.from_numpy(flat0).to(dev, torch.float64)
    s_ref = [torch.full_like(p_ref, spec.slot_init(i)) for i in range(spec.num_slots)]
    p_max = p_ref.abs()
    for k, g in enumerate(grads):
        apply_update(spec, p_ref, torch.from_numpy(g).to(dev, torch.float64), s_ref, k + 1)
        p_max = torch.maximum(p_max, p_ref.abs())
    p_ref, p_max, s_ref = p_ref.cpu(), p_max.cpu(), [t.cpu() for t in s_ref]
    got_p = lay.flatten(master.weights())
    got_s = [lay.flatten(s) for s in master.slot_arrays()]
    tag = f"{opt}/{model}/{master_kind} max_batch={max_batch}"
    err_p, ratio_p = _within(f"{tag} parameters", got_p[valid], p_ref.numpy()[valid], 2e-6)
    atol = [2e-6] * len(s_ref)
    if opt == "ftrl":
        # the linear slot accumulates sigma * p with sigma = (sqrt(n + g^2) - sqrt(n)) / lr: the fp32 difference of the
        # square roots is exact only to a few ulp of sqrt(n), so its error is a few ulp of sqrt(n) / lr * |p| per step
        # (measured 3.3e-6 on 2 of 269k elements where that scale is ~30)
        atol[1] = 2e-6 + 8 * 2.0 ** -23 * (s_ref[0].sqrt() / spec.hyper["lr"] * p_max).numpy()[valid]
    slot_errs = [_within(f"{tag} slot {i}", a[valid], b.numpy()[valid], atol[i]) for i, (a, b) in enumerate(zip(got_s, s_ref))]
    print(f"[applier] {tag}: parameters max-abs {err_p:.2e} ({ratio_p:.2f}x tolerance); slots "
          + (", ".join(f"max-abs {e:.2e} ({r:.2f}x)" for e, r in slot_errs) or "none"))
    if spec.hyper.get("l1", 0.0) > 0:
        assert (p_ref.numpy()[quiet] == 0).all()
        assert (got_p[quiet] == 0).all(), f"{opt}: {int((got_p[quiet] != 0).sum())} clamped parameters are not exactly 0"
    # published bf16 operands are the bf16 image of the final fp32 parameters, bit for bit
    pub = torch.from_numpy(lay.publish_reference(got_p)).to(torch.bfloat16)
    shadows = [master.shadow] if master_kind == "served" else [master.view("shadow", r, dev) for r in range(master.n)]
    for sh in shadows:
        assert torch.equal(sh.cpu(), pub)
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


def test_fused_dropout_mask_statistics():
    """K13: tf.nn.dropout after a dense layer runs inside the compiled plan (Philox mask in the GEMM epilogue).  The
    statistics of the mask recovered from the stored activation (reference semantics: keep with prob p, scale by 1/p -
    tf.nn.dropout; ml_util.py:70-71).  The exact mask and the gradients are checked in test_gpu_dropout.py."""
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
    master.close()
