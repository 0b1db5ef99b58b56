"""Locked push with a replica_version word: the write-lock grant and the first tile's master-tuple loads run before the
push waits for the step's last GEMM, and the loads are reused when SF_CTRL_VERSION, read under the lock, still equals
the version of the worker's own last push.  Otherwise (first push, another worker's push, a host write of the master
state) the push reloads them; word 6 of the worker's push sync words counts those reloads."""
import numpy as np
import pytest
import torch

from push_helpers import wait_pushes
from sparkflow_b200.ops import native
from sparkflow_b200.ops.optimizers import OptimizerSpec
from test_gpu_pull_elision import B, NAME, _assert_replica_current, _engine, _pull, _second_worker
from test_step_gradients import DEV, UPDATE_TOL, _data, _model, _weights, _worker, oracle

# a large epsilon keeps the Adam update linear in small gradients, so the float64 comparison of the production steps is
# not dominated by the sign of gradients within rounding of zero
ADAM = ("adam", dict(learning_rate=0.01, epsilon=0.1))


def _reloads(worker):
    return int(worker.sync_push[6])


def _grad(worker, seed):
    """fill the worker's gradient buffer with a seeded gradient"""
    g = torch.from_numpy(np.random.default_rng(seed).standard_normal(worker.layout.total).astype(np.float32) * 0.1)
    worker.grads.copy_(g.to(DEV))
    torch.cuda.synchronize()


def _push(worker, drop=0):
    """the worker's push kernel with the arguments of its step plans"""
    loss_out = torch.zeros(2, device=DEV)
    worker.C.push(worker._push_args(loss_out, drop=drop), native.ptr(worker.sync_push), 0, native.current_stream())
    torch.cuda.synchronize()
    assert worker.C.read_error_code() == 0


def _snapshot(master):
    torch.cuda.synchronize()
    return master.state.clone(), master.shadow.clone(), master.ctrl.clone()


def _restore(master, snap):
    state, shadow, ctrl = snap
    master.state.copy_(state)
    master.shadow.copy_(shadow)
    master.ctrl.copy_(ctrl)
    torch.cuda.synchronize()


def _assert_same(tag, a, b):
    for name, x, y in zip(("state", "publish"), a[:2], b[:2]):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x.view(torch.int16),
                           y.view(torch.int32) if y.dtype == torch.float32 else y.view(torch.int16)), f"{tag}: {name} differs"


@pytest.mark.gpu
def test_production_steps_reuse_the_early_loads():
    """One worker, lock mode, Adam, six production steps: only the first push reloads its tuples; the master's
    parameters and slots track the host parameter server fed the float64 oracle's gradients, and the replica is the
    master's publish bit for bit after every step."""
    from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer

    _, lp, _ = _model(NAME)
    spec = OptimizerSpec.from_tf_kwargs(*ADAM)
    w0 = _weights(NAME)
    X, Y = _data(NAME, 2 * B + 7, seed=B + 5)
    master, worker = _worker(NAME, w0, spec, lock=True)
    try:
        assert worker.own_publish
        eng = _engine(worker, X, Y)
        server = ParameterServer(w0, spec)
        ref = LocalTransport(server)
        rng = np.random.default_rng(11)
        steps = [slice(0, B), slice(B, 2 * B), rng.permutation(2 * B + 7)[:B], slice(7, B + 7), slice(0, B), rng.permutation(2 * B + 7)[:B]]
        for k, rows in enumerate(steps):
            w_k = master.weights()
            eng.train(rows, pull=True)
            eng.finish()
            ref.push(oracle(lp, w_k, X[rows], Y[rows], emulate_bf16=True)[1])
            tag = f"step {k}"
            _assert_replica_current(tag, master, worker)
            assert _reloads(worker) == 1, f"{tag}: {_reloads(worker)} pushes reloaded their tuples (only the first should)"
            assert int(worker.replica_version[0]) == int(master.ctrl[1]) == k + 1, tag
        assert wait_pushes(master, len(steps)) == len(steps)
        got = [master.weights()] + master.slot_arrays()
        want = [ref.pull()] + server.slot_arrays()
        for col, (g_col, r_col) in enumerate(zip(got, want)):
            for a, b, a0, v in zip(g_col, r_col, w0 if col == 0 else [None] * len(g_col), lp.var_order):
                du, dr = (a - a0, b - a0) if col == 0 else (a, b)
                err = np.linalg.norm(du - dr) / np.linalg.norm(dr)
                assert np.isfinite(du).all() and err <= UPDATE_TOL, f"{v} (column {col}): off by {err:.2e}"
    finally:
        master.close()


@pytest.mark.gpu
def test_early_loads_and_reload_agree_bitwise():
    """The same push from the same master state and gradient, once with valid early loads and once forced to reload
    (replica_version = -1): master state, publish and replica are bit-identical."""
    spec = OptimizerSpec.from_tf_kwargs(*ADAM)
    master, worker = _worker(NAME, _weights(NAME), spec, lock=True)
    try:
        _grad(worker, 0)
        _push(worker)                               # the first push: no version yet, reloads
        assert _reloads(worker) == 1 and int(worker.replica_version[0]) == 1
        before = _snapshot(master)
        replica = worker.replica.clone()
        _grad(worker, 1)
        _push(worker)
        assert _reloads(worker) == 1, "a push right after the worker's own push reloaded"
        early = _snapshot(master) + (worker.replica.clone(),)

        _restore(master, before)
        worker.replica.copy_(replica)
        worker.replica_version.fill_(-1)
        _grad(worker, 1)
        _push(worker)
        assert _reloads(worker) == 2, "a push with replica_version -1 used its early loads"
        reload = _snapshot(master) + (worker.replica.clone(),)
        _assert_same("early vs reload", early, reload)
        assert torch.equal(early[3], reload[3]), "replica differs"
        assert torch.equal(early[2], reload[2]), "control block differs"
        _assert_replica_current("after the reload", master, worker)
    finally:
        master.close()


@pytest.mark.gpu
def test_interleaved_workers_reload_after_each_others_push():
    """Two workers on one master push A, B, A, A, B, A, B (dropped), A: a push after the other worker's applied push
    reloads, a push after the worker's own push or after the other's dropped push does not; the master ends where one
    worker applying the same gradients in the same order ends."""
    spec = OptimizerSpec.from_tf_kwargs(*ADAM)
    w0 = _weights(NAME)
    order = [("a", 0), ("b", 0), ("a", 0), ("a", 0), ("b", 0), ("a", 0), ("b", 1), ("a", 0)]
    expect = {"a": [1, 2, 2, 3, 3], "b": [1, 2, 2]}       # reload count of each worker after each of its pushes
    master, a = _worker(NAME, w0, spec, lock=True)
    try:
        b = _second_worker(master)
        workers, seen = {"a": a, "b": b}, {"a": [], "b": []}
        for k, (who, drop) in enumerate(order):
            w = workers[who]
            _grad(w, 100 + k)
            _push(w, drop=drop)
            seen[who].append(_reloads(w))
            if not drop:
                _assert_replica_current(f"push {k} ({who})", master, w)
        assert seen == expect, seen
        c = master.counters()
        assert c["pushes"] == 7 and c["dropped"] == 1 and c["lock"] == 0, c
        got = _snapshot(master)

        ref_master, r = _worker(NAME, w0, spec, lock=True)
        try:
            for k, (who, drop) in enumerate(order):
                if not drop:
                    _grad(r, 100 + k)
                    _push(r)
            assert _reloads(r) == 1
            _assert_same("two workers vs one", got, _snapshot(ref_master))
        finally:
            ref_master.close()
    finally:
        master.close()


def _twin(master, spec):
    """a second master holding a copy of ``master``'s state, and its worker (no version yet: its first push reloads)"""
    twin, w = _worker(NAME, _weights(NAME), spec, lock=True)
    _restore(twin, _snapshot(master))
    return twin, w


@pytest.mark.gpu
@pytest.mark.parametrize("write", ["load_slots", "load_weights"])
def test_host_write_makes_the_next_push_reload(write):
    """After a host write of the master state between two pushes of one worker, the next push reloads and applies to
    the written state (bit for bit what a push that reloads from a copy of that state computes); after load_weights a
    pull copies."""
    spec = OptimizerSpec.from_tf_kwargs(*ADAM)
    master, worker = _worker(NAME, _weights(NAME), spec, lock=True)
    try:
        for k in range(2):
            _grad(worker, 200 + k)
            _push(worker)
        assert _reloads(worker) == 1
        version = int(master.ctrl[1])
        rng = np.random.default_rng(5)
        if write == "load_slots":
            master.load_slots([[np.abs(rng.standard_normal(s.shape)).astype(np.float32) * 0.01 for s in master.weights()]
                               for _ in range(spec.num_slots)], step=40)
        else:
            master.load_weights(_weights(NAME, seed=3))
            assert _pull(worker), "the pull after load_weights skipped the copy"
        assert int(master.ctrl[1]) == version + 1, "the host write did not move the version on"
        twin, tw = _twin(master, spec)
        try:
            _grad(worker, 300)
            _push(worker)
            assert _reloads(worker) == 2, f"the push after {write} used its early loads"
            _grad(tw, 300)
            _push(tw)
            _assert_same(f"after {write}", _snapshot(master), _snapshot(twin))
        finally:
            twin.close()
    finally:
        master.close()
