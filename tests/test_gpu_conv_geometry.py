"""SAME-padded / strided convolutions and general max-pools on the native path: every new or generalized kernel against
PyTorch fp32, the compiled training step of the new zoo CNNs against the interpreter oracle, sessions and inference on
them, and the unchanged kernel sequence of the VALID stride-1 ``cnn`` model."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from kernel_usage import needs_binary_utils, res_usage
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import compile_graph, conv_geometry
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout, round_up
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs
from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer
from sparkflow_b200.parallel.worker import B200Engine, TorchEngine

ACT = {None: 0, "relu": 1, "sigmoid": 2, "tanh": 3}


def _act(x, a):
    return {None: lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[a](x)


def _dact(a_out, a):
    if a == "relu":
        return (a_out > 0).float()
    if a == "sigmoid":
        return a_out * (1 - a_out)
    if a == "tanh":
        return 1 - a_out * a_out
    return torch.ones_like(a_out)


@pytest.fixture(scope="module")
def C():
    return native.cuda_ext()


def _geometry(h, w, kh, kw, sh, sw, padding):
    oh, pt, pb = conv_geometry(h, kh, sh, padding)
    ow, pl, pr = conv_geometry(w, kw, sw, padding)
    return oh, ow, (pt, pb, pl, pr)


def _nchw_pad(x_nhwc, pads, value=0.0):
    pt, pb, pl, pr = pads
    return F.pad(x_nhwc.float().permute(0, 3, 1, 2), (pl, pr, pt, pb), value=value)


# (padding, stride, odd / even size, cin: 1 = scalar kernels, 32 = vec8 kernels)
GEOMS = [(p, s, h, c) for p in ("VALID", "SAME") for s in (1, 2) for h in (9, 10) for c in (1, 32)]


@pytest.mark.parametrize("padding,stride,h,cin", GEOMS)
def test_im2col_col2im_geometry(C, padding, stride, h, cin):
    n, w, kh, kw = 3, h + 3, 3, 3
    oh, ow, pads = _geometry(h, w, kh, kw, stride, stride, padding)
    g = torch.Generator(device="cuda").manual_seed(h * 100 + cin + stride)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(torch.bfloat16)
    M, K = n * oh * ow, kh * kw * cin
    ldK, ldM = round_up(K, 8), round_up(M, 8)
    ref = F.unfold(_nchw_pad(x, pads), (kh, kw), stride=stride)                       # [n, c*kh*kw, L] in (c, kh, kw) order
    ref = ref.reshape(n, cin, kh * kw, oh * ow).permute(0, 3, 2, 1).reshape(M, K)     # -> (kh, kw, c) order
    st = native.current_stream()
    geo = dict(sh=stride, sw=stride, pad_top=pads[0], pad_left=pads[2], out_h=oh, out_w=ow)
    # with the transposed copy (scalar tile kernel) and without it (vec8 kernel when cin % 8 == 0)
    for want_t in (True, False):
        out = torch.full((M, ldK), 7.0, dtype=torch.bfloat16, device="cuda")
        outT = torch.zeros(K, ldM, dtype=torch.bfloat16, device="cuda") if want_t else None
        C.im2col(native.ptr(x), n, h, w, cin, kh, kw, native.ptr(out), ldK, native.ptr(outT), ldM if want_t else 0, st, **geo)
        torch.cuda.synchronize()
        assert torch.equal(out[:, :K].float(), ref)
        assert torch.all(out[:, K:] == 0)
        if want_t:
            assert torch.equal(outT[:, :M].float().t(), ref)
    # col2im == adjoint of im2col (fold over the padded image, then crop the border)
    dcols = torch.randn(M, ldK, device="cuda", generator=g).to(torch.bfloat16)
    din = torch.zeros(n, h, w, cin, dtype=torch.bfloat16, device="cuda")
    C.col2im(native.ptr(dcols), ldK, n, h, w, cin, kh, kw, native.ptr(din), st, **geo)
    torch.cuda.synchronize()
    d = dcols[:, :K].float().reshape(n, oh * ow, kh * kw, cin).permute(0, 3, 2, 1).reshape(n, cin * kh * kw, oh * ow)
    pt, pb, pl, pr = pads
    full = F.fold(d, (h + pt + pb, w + pl + pr), (kh, kw), stride=stride)
    ref_in = full[:, :, pt:pt + h, pl:pl + w].permute(0, 2, 3, 1)
    torch.testing.assert_close(din.float(), ref_in, rtol=2e-2, atol=5e-2)


POOLS = [(k, s, p, h, c) for (k, s) in ((3, 2), (2, 2), (3, 1), (4, 3)) for p in ("VALID", "SAME") for h in (9, 10) for c in (8, 32)]


@pytest.mark.parametrize("k,stride,padding,h,c", POOLS)
def test_general_maxpool_fwd_bwd(C, k, stride, padding, h, c):
    n, w = 3, h + 1
    oh, ow, pads = _geometry(h, w, k, k, stride, stride, padding)
    g = torch.Generator(device="cuda").manual_seed(k * 1000 + h * 10 + c)
    a = torch.tanh(torch.randn(n, h, w, c, device="cuda", generator=g)).to(torch.bfloat16)      # conv output after tanh
    out = torch.zeros(n, oh, ow, c, dtype=torch.bfloat16, device="cuda")
    am = torch.full((n, oh, ow, c), 255, dtype=torch.uint8, device="cuda")
    st = native.current_stream()
    C.maxpool_gen_fwd(native.ptr(a), n, h, w, c, k, k, stride, stride, pads[0], pads[2], oh, ow, native.ptr(out), native.ptr(am), st)
    torch.cuda.synchronize()
    af = a.float().permute(0, 3, 1, 2).requires_grad_(True)
    ref = F.max_pool2d(F.pad(af, (pads[2], pads[3], pads[0], pads[1]), value=float("-inf")), k, stride)
    assert torch.equal(out.float(), ref.detach().permute(0, 2, 3, 1))
    # the stored in-window index points at a real cell holding the maximum
    assert int(am.max()) < k * k
    dy, dx = am.long() // k, am.long() % k
    ys = (torch.arange(oh, device="cuda") * stride - pads[0]).view(1, oh, 1, 1) + dy
    xs = (torch.arange(ow, device="cuda") * stride - pads[2]).view(1, 1, ow, 1) + dx
    assert bool(((ys >= 0) & (ys < h) & (xs >= 0) & (xs < w)).all())
    bi = torch.arange(n, device="cuda").view(n, 1, 1, 1).expand_as(ys)
    ci = torch.arange(c, device="cuda").view(1, 1, 1, c).expand_as(ys)
    assert torch.equal(a[bi, ys, xs, ci], out)
    # backward: gather of every window a position won, times tanh'(a), and the bias gradient
    dout = torch.randn(n, oh, ow, c, device="cuda", generator=g).to(torch.bfloat16)
    M = n * h * w
    dz = torch.full((M, c), 7.0, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(c, device="cuda")
    C.maxpool_gen_bwd(native.ptr(dout), native.ptr(am), n, h, w, c, k, k, stride, stride, pads[0], pads[2], oh, ow, native.ptr(a),
                      ACT["tanh"], native.ptr(dz), c, native.ptr(db), st)
    torch.cuda.synchronize()
    scat = torch.zeros(n, h, w, c, device="cuda").index_put_((bi, ys, xs, ci), dout.float(), accumulate=True)
    exp = (scat * _dact(a.float(), "tanh")).reshape(M, c)
    torch.testing.assert_close(dz.float(), exp, rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(db, exp.sum(0), rtol=1e-2, atol=5e-2)
    # ... and autograd through the -inf padded max-pool agrees wherever the window had a unique winner
    ref.backward(dout.float().permute(0, 3, 1, 2))
    auto = (af.grad.permute(0, 2, 3, 1) * _dact(a.float(), "tanh")).reshape(M, c)
    torch.testing.assert_close(dz.float().sum(), auto.sum(), rtol=1e-2, atol=2e-1)
    assert (dz.float() - auto).abs().gt(2e-2).float().mean().item() < 0.02


@pytest.mark.parametrize("act", ["relu", "sigmoid", "tanh"])
@pytest.mark.parametrize("M,c", [(1000, 32), (4 * 7 * 7, 64), (37, 16)])
def test_act_bwd_bias(C, act, M, c):
    g = torch.Generator(device="cuda").manual_seed(M + c)
    a = _act(torch.randn(M, c, device="cuda", generator=g), act).to(torch.bfloat16)
    grad = torch.randn(M, c, device="cuda", generator=g).to(torch.bfloat16)
    dz = torch.full((M, c), 7.0, dtype=torch.bfloat16, device="cuda")
    db = torch.full((c,), 1.0, device="cuda")
    C.act_bwd_bias(native.ptr(grad), c, M, c, native.ptr(a), ACT[act], native.ptr(dz), c, native.ptr(db), native.current_stream())
    torch.cuda.synchronize()
    exp = grad.float() * _dact(a.float(), act)
    torch.testing.assert_close(dz.float(), exp, rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(db - 1.0, exp.sum(0), rtol=1e-2, atol=5e-2)       # accumulates into the bias gradient


@pytest.mark.parametrize("n,h,w,cin,kh,kw,cout,act", [(5, 28, 28, 1, 5, 5, 32, "relu"), (3, 12, 12, 3, 3, 3, 16, "tanh"),
                                                       (2, 10, 10, 2, 3, 3, 8, None), (2, 14, 14, 1, 3, 3, 64, "sigmoid")])
def test_conv_first_fused_same_padding(C, n, h, w, cin, kh, kw, cout, act):
    """Fused first conv (stride 1, SAME) + bias + activation + 2x2 max-pool, and its weight / bias gradient, against torch."""
    oh, ow, pads = _geometry(h, w, kh, kw, 1, 1, "SAME")
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(torch.bfloat16)
    K = kh * kw * cin
    wmat = (torch.randn(K, cout, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    ld_w = round_up(K, 8)
    wT = torch.zeros(cout, ld_w, dtype=torch.bfloat16, device="cuda")
    wT[:, :K] = wmat.t()
    bias = torch.randn(cout, device="cuda", generator=g) * 0.1
    ph, pw = oh // 2, ow // 2
    pooled = torch.zeros(n, ph, pw, cout, dtype=torch.bfloat16, device="cuda")
    argmax = torch.zeros(n, ph, pw, cout, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    geo = dict(pad_top=pads[0], pad_left=pads[2], out_h=oh, out_w=ow)
    C.conv_first_fwd(x.data_ptr(), n, h, w, cin, kh, kw, cout, wT.data_ptr(), ld_w, bias.data_ptr(), ACT[act], pooled.data_ptr(),
                     argmax.data_ptr(), st, **geo)
    torch.cuda.synchronize()
    xt = _nchw_pad(x, pads)
    wt = wmat.float().reshape(kh, kw, cin, cout).permute(3, 2, 0, 1).clone().requires_grad_(True)
    bt = bias.clone().requires_grad_(True)
    conv = _act(F.conv2d(xt, wt, bt), act)
    assert conv.shape[2:] == (oh, ow)
    ref = F.max_pool2d(conv, 2)
    assert torch.allclose(pooled.float().permute(0, 3, 1, 2), ref, rtol=2e-2, atol=2e-2)
    gp = torch.randn(n, ph, pw, cout, device="cuda", generator=g).to(torch.bfloat16)
    dW = torch.zeros(K, cout, device="cuda")
    db = torch.zeros(cout, device="cuda")
    C.conv_first_wgrad(x.data_ptr(), n, h, w, cin, kh, kw, cout, gp.data_ptr(), pooled.data_ptr(), argmax.data_ptr(), ACT[act], dW.data_ptr(),
                       db.data_ptr(), st, **geo)
    torch.cuda.synchronize()
    am = argmax.long().permute(0, 3, 1, 2)
    ys = 2 * torch.arange(ph, device="cuda").view(1, 1, ph, 1) + am // 2
    xs = 2 * torch.arange(pw, device="cuda").view(1, 1, 1, pw) + am % 2
    picked = conv[torch.arange(n, device="cuda").view(n, 1, 1, 1), torch.arange(cout, device="cuda").view(1, cout, 1, 1), ys, xs]
    (picked * gp.float().permute(0, 3, 1, 2)).sum().backward()
    ref_dW = wt.grad.permute(2, 3, 1, 0).reshape(K, cout)
    scale = max(1.0, ref_dW.abs().max().item())
    assert (dW - ref_dW).abs().max().item() < 3e-2 * scale
    assert torch.allclose(db, bt.grad, rtol=3e-2, atol=3e-2 * max(1.0, bt.grad.abs().max().item()))


@needs_binary_utils
def test_new_and_generalized_kernels_have_no_stack_frame():
    use = {k: s for k, (_, s) in res_usage().items()}
    want = [k for k in use if re.match(r"sf::(maxpool_gen_fwd_kernel|maxpool_gen_bwd_kernel|act_bwd_bias_kernel|im2col_kernel|im2col_vec8_kernel|"
                                        r"col2im_kernel|col2im_vec8_kernel|conv_first_fwd_kernel|conv_first_wgrad_kernel)", k)]
    assert len(want) >= 15, sorted(use)[:10]
    assert not {k: use[k] for k in want if use[k] != 0}


# ------------------------------------------------------------------------------------------------------------------------
# engine level
# ------------------------------------------------------------------------------------------------------------------------
def _data(n, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.random((n, 784), dtype=np.float32)
    Y = np.eye(10, dtype=np.float32)[rng.integers(0, 10, n)]
    return X, Y


def _worker(name, spec, lock):
    ir = GraphIR.from_metagraph(zoo.build(name))
    lp = compile_graph(ir, "x:0", "y:0")
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    master = MasterState(lay, spec, torch.device("cuda:0"))
    w0 = GraphProgram(ir).init_weights(seed=1)
    master.load_weights(w0)
    worker = DeviceWorker(ir, "x:0", "y:0", spec, master, acquire_lock=lock, shared=False)
    return ir, master, worker, w0


@pytest.mark.parametrize("name", ["cnn_same", "cnn_strided"])
@pytest.mark.parametrize("lock", [False, True])
def test_compiled_step_tracks_oracle_new_geometry(name, lock):
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    ir, master, worker, w0 = _worker(name, spec, lock)
    X, Y = _data(256)
    eng = B200Engine(worker)
    eng.load_partition(X, Y)
    ps = ParameterServer(w0, spec, acquire_lock=lock)
    ref = TorchEngine(ir, "x:0", "y:0", LocalTransport(ps))
    ref.load_partition(X, Y)
    rows = [slice(0, 64), slice(64, 128), np.arange(100, 164), slice(192, 256), slice(0, 64)]
    for r in rows:
        eng.train(r, pull=True)
        ref.train(r, pull=True)
    eng.finish()
    got, exp = master.weights(), ps.weights()
    for a, b, v in zip(got, exp, ir.trainable):
        assert np.abs(a - b).max() < 5 * 0.001 * len(rows), v.name
        assert np.mean(np.abs(a - b)) < 0.35 * 0.001 * len(rows), v.name
    cnt = master.counters()
    assert cnt["pushes"] == len(rows) and cnt["lock"] == 0
    loss_gpu = worker.partition_loss(eng.X, eng.Y)
    loss_ref = GraphProgram(ir).loss(ref._feed(slice(0, 256)), got)
    assert abs(loss_gpu - loss_ref) < 2e-2 * max(1.0, abs(loss_ref))
    names = worker.last_plan_names() if hasattr(worker, "last_plan_names") else []
    if name == "cnn_strided":
        assert "maxpool_gen_fwd" in names and "maxpool_gen_bwd" in names and names.count("act_bwd_bias") == 2, names
    master.close()


def test_session_trains_cnn_strided_natively():
    from sparkflow_b200.parallel.session import TrainingSession

    rng = np.random.default_rng(3)
    centers = rng.random((10, 784), dtype=np.float32)
    lab = rng.integers(0, 10, 1200)
    X = np.clip(centers[lab] + 0.1 * rng.normal(0, 1, (1200, 784)), 0, 1).astype(np.float32)
    Y = np.eye(10, dtype=np.float32)[lab]
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.002))
    sess = TrainingSession(zoo.build("cnn_strided"), "x:0", "y:0", spec, acquire_lock=True, engine="b200", seed=0, devices=[0]).open()
    try:
        assert sess.engine_kind == "b200"
        eng = sess.make_engine(torch.device("cuda", 0))
        eng.load_partition(X, Y)
        l0 = eng.partition_loss()
        for k in range(16):
            eng.train(slice((k % 4) * 300, (k % 4) * 300 + 300), pull=True)
        eng.finish()
        l1 = eng.partition_loss()
        assert np.isfinite(l1) and l1 < 0.8 * l0, (l0, l1)
        assert sess.counters()["pushes"] == 16
    finally:
        sess.close()


def test_inference_on_cnn_same_runs_the_compiled_forward_plan(monkeypatch):
    from sparkflow_b200.ml_util import run_inference

    graph = zoo.build("cnn_same")
    ir = GraphIR.from_metagraph(graph)
    lp = compile_graph(ir, "x:0", "y:0")
    logits = lp.layers[-1].tensors["bias"]                     # tfOutput = the last dense layer's output
    w = GraphProgram(ir).init_weights(seed=4)
    w = [a if a.ndim > 1 else (0.05 * np.random.default_rng(2).standard_normal(a.shape)).astype(np.float32) for a in w]
    X, _ = _data(300, seed=9)
    ref = GraphProgram(ir, "cuda").forward(logits, {"x:0": X}, w).detach().cpu().numpy()

    def no_interpreter(*a, **k):
        raise AssertionError("prediction fell back to the interpreter")

    monkeypatch.setattr(GraphProgram, "forward", no_interpreter)
    got = run_inference(graph, w, X, "x:0", logits)
    assert got.shape == ref.shape == (300, 10)
    assert np.abs(got - ref).max() < 3e-2 * max(1.0, np.abs(ref).max()), np.abs(got - ref).max()
    pred = run_inference(graph, w, X, "x:0", "out:0")
    assert (pred.astype(np.int64) == ref.argmax(1)).mean() > 0.9


# kernel sequences of the VALID stride-1 cnn model's plans (batch 64, lock and Hogwild alike), recorded on the code before
# SAME / strided geometry existed
CNN_TRAIN_NAMES = ["pull@1", "cast_transpose", "conv_first_fwd", "im2col", "conv3", "maxpool_fwd", "fwd6+loss", "wgrad6@2"] + \
                  ["dgrad6", "maxpool_bwd", "wgrad3@1", "dgrad3", "col2im", "conv_first_wgrad", "push"]
CNN_FORWARD_NAMES = ["pull", "cast_transpose", "conv_first_fwd", "im2col", "conv3", "maxpool_fwd", "fwd6", "argmax"]


def test_cnn_plans_issue_the_same_kernels():
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    for lock in (False, True):
        ir, master, worker, w0 = _worker("cnn", spec, lock)
        plan, _ = worker.build_plan(64, 0, with_pull=True, with_push=True)
        assert list(plan.names()) == CNN_TRAIN_NAMES
        fplan, _ = worker.build_forward_plan(64, post="ArgMax", with_pull=True)
        assert list(fplan.names()) == CNN_FORWARD_NAMES
        master.close()
