"""Numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout, round_up
from sparkflow_b200.ops.optimizers import OPT_IDS, OptimizerSpec, apply_update, init_slots
from push_helpers import OPTIMIZERS

ACT = {None: 0, "relu": 1, "sigmoid": 2, "tanh": 3}


def _act(x, a):
    return {None: lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[a](x)


@pytest.fixture(scope="module")
def C():
    return native.cuda_ext()


def test_cast_transpose(C):
    x = torch.randn(300, 784, device="cuda")
    ld, ldt = round_up(784, 8), round_up(300, 8)
    out = torch.full((300, ld), 9.0, dtype=torch.bfloat16, device="cuda")
    outT = torch.full((784, ldt), 9.0, dtype=torch.bfloat16, device="cuda")
    C.cast_transpose(native.ptr(x), 784, 0, native.ptr(out), ld, native.ptr(outT), ldt, 300, 784,
                     native.current_stream())
    torch.cuda.synchronize()
    assert torch.equal(out[:, :784], x.to(torch.bfloat16))
    assert torch.equal(outT[:, :300], x.to(torch.bfloat16).t())
    assert torch.all(outT[:, 300:] == 0)
    idx = torch.randperm(300, device="cuda", dtype=torch.int32)[:128].contiguous()
    out2 = torch.zeros(128, ld, dtype=torch.bfloat16, device="cuda")
    C.cast_transpose(native.ptr(x), 784, native.ptr(idx), native.ptr(out2), ld, 0, 0, 128, 784,
                     native.current_stream())
    torch.cuda.synchronize()
    assert torch.equal(out2[:, :784], x[idx.long()].to(torch.bfloat16))


@pytest.mark.parametrize("B,Cc", [(300, 10), (64, 1000), (7, 3)])
def test_softmax_xent(C, B, Cc):
    z = torch.randn(B, Cc, device="cuda") * 3
    y = torch.nn.functional.one_hot(torch.randint(0, Cc, (B,), device="cuda"), Cc).float()
    ld, ldt = round_up(Cc, 8), round_up(B, 8)
    loss = torch.zeros(1, device="cuda")
    dz = torch.full((B, ld), 5.0, dtype=torch.bfloat16, device="cuda")
    dzT = torch.zeros(Cc, ldt, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(Cc, device="cuda")
    C.softmax_xent(native.ptr(z), Cc, native.ptr(y), Cc, native.ptr(loss), native.ptr(dz), ld, native.ptr(dzT), ldt,
                   native.ptr(db), B, Cc, native.current_stream())
    torch.cuda.synchronize()
    zr = z.clone().requires_grad_(True)
    ref = -(y * torch.log_softmax(zr, 1)).sum(1).mean()
    ref.backward()
    torch.testing.assert_close(loss[0], ref.detach(), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dz[:, :Cc].float(), zr.grad, rtol=2e-2, atol=1e-4)
    torch.testing.assert_close(dzT[:, :B].float().t(), zr.grad, rtol=2e-2, atol=1e-4)
    assert torch.all(dz[:, Cc:] == 0)
    torch.testing.assert_close(db, zr.grad.sum(0), rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize("act", [None, "sigmoid"])
def test_mse(C, act):
    B, Cc = 256, 784
    pre = torch.randn(B, Cc, device="cuda", requires_grad=True)
    out = _act(pre, act)
    tgt = torch.rand(B, Cc, device="cuda")
    ref = ((out - tgt) ** 2).mean()
    ref.backward()
    ld, ldt = round_up(Cc, 8), round_up(B, 8)
    loss = torch.zeros(1, device="cuda")
    dz = torch.zeros(B, ld, dtype=torch.bfloat16, device="cuda")
    dzT = torch.zeros(Cc, ldt, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(Cc, device="cuda")
    o = out.detach().contiguous()
    C.mse_loss(native.ptr(o), Cc, native.ptr(tgt), Cc, ACT[act], native.ptr(loss), native.ptr(dz), ld,
               native.ptr(dzT), ldt, native.ptr(db), B, Cc, native.current_stream())
    torch.cuda.synchronize()
    torch.testing.assert_close(loss[0], ref.detach(), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(dz[:, :Cc].float(), pre.grad, rtol=2e-2, atol=1e-7)
    torch.testing.assert_close(dzT[:, :B].float().t(), pre.grad, rtol=2e-2, atol=1e-7)
    torch.testing.assert_close(db, pre.grad.sum(0), rtol=1e-3, atol=1e-7)


def test_argmax(C):
    z = torch.randn(333, 10, device="cuda")
    out = torch.zeros(333, device="cuda")
    C.argmax_rows(native.ptr(z), 10, native.ptr(out), 333, 10, native.current_stream())
    torch.cuda.synchronize()
    assert torch.equal(out.long(), z.argmax(1))


SHAPES = [("dense/kernel", (784, 256)), ("dense/bias", (256,)), ("dense_1/kernel", (256, 256)),
          ("dense_1/bias", (256,)), ("dense_2/kernel", (256, 10)), ("dense_2/bias", (10,))]


def _push_setup(C, spec, lock_mode=0):
    lay = ParamLayout.build(SHAPES)
    dev = "cuda"
    state = torch.zeros(lay.total, 4, device=dev)
    mask = torch.from_numpy(lay.valid_mask()).to(dev)
    state[mask, 0] = torch.randn(int(mask.sum()), device=dev) * 0.1
    for i in range(spec.num_slots):
        state[:, 1 + i] = spec.slot_init(i)
    p = state[:, 0]
    slots = [state[:, 1 + i] for i in range(spec.num_slots)] + [None] * (3 - spec.num_slots)
    ctrl = torch.zeros(C.CTRL_WORDS, dtype=torch.int32, device=dev)
    shadow = torch.zeros(lay.shadow_total, dtype=torch.bfloat16, device=dev)
    grad = torch.zeros(lay.total, device=dev)
    segs = torch.frombuffer(bytearray(C.pack_segs(lay.seg_rows())), dtype=torch.uint8).to(dev)
    tmap = torch.from_numpy(lay.tile_map()).to(dev)
    lsync = torch.zeros(8, dtype=torch.int32, device=dev)
    loss_acc = torch.zeros(1, device=dev)
    loss_out = torch.zeros(1, device=dev)
    args = dict(state=native.ptr(state), ctrl=native.ptr(ctrl), shadow_dst=[native.ptr(shadow)], grad=native.ptr(grad),
                loss_acc=native.ptr(loss_acc), loss_out=native.ptr(loss_out), segs=native.ptr(segs),
                tile_map=native.ptr(tmap), num_tiles=int(tmap.shape[0]), optimizer=spec.opt_id,
                lock_mode=lock_mode, grad_scale=1.0, hyper=spec.native_hyper())
    keep = dict(lay=lay, state=state, p=p, slots=slots, ctrl=ctrl, shadow=shadow, grad=grad, segs=segs, tmap=tmap, lsync=lsync,
                loss_acc=loss_acc, loss_out=loss_out, mask=mask)
    return args, keep


@pytest.mark.parametrize("name,kw", OPTIMIZERS)
@pytest.mark.parametrize("lock_mode", [0, 1])
def test_push_matches_reference_optimizer(C, name, kw, lock_mode):
    spec = OptimizerSpec.from_tf_kwargs(name, kw)
    args, k = _push_setup(C, spec, lock_mode)
    p_ref = k["p"].clone().contiguous()
    s_ref = [s.clone().contiguous() for s in k["slots"] if s is not None]
    for step in range(1, 4):
        g = torch.zeros_like(k["grad"])
        g[k["mask"]] = torch.randn(int(k["mask"].sum()), device="cuda") * 0.05
        k["grad"].copy_(g)
        k["loss_acc"].fill_(float(step))
        C.push(args, native.ptr(k["lsync"]), 0, native.current_stream())
        torch.cuda.synchronize()
        assert C.read_error_code() == 0
        apply_update(spec, p_ref, g, s_ref, step)
        torch.testing.assert_close(k["p"][k["mask"]], p_ref[k["mask"]], rtol=2e-4, atol=2e-6)
        for a, b in zip([s for s in k["slots"] if s is not None], s_ref):
            torch.testing.assert_close(a[k["mask"]], b[k["mask"]], rtol=2e-4, atol=1e-6)
        assert torch.all(k["grad"] == 0), "push must consume (zero) the gradient buffer"
        assert float(k["loss_out"][0]) == float(step) and float(k["loss_acc"][0]) == 0.0
        ctrl = k["ctrl"].cpu().numpy()
        assert ctrl[0] == 0 and ctrl[1] == step and ctrl[2] == step and ctrl[3] == step
    exp = torch.from_numpy(k["lay"].publish_reference(k["p"].contiguous().cpu().numpy())).to(torch.bfloat16)
    assert torch.equal(k["shadow"].cpu(), exp)


def test_push_drop_fault_injection(C):
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.01))
    args, k = _push_setup(C, spec)
    args["drop"] = 1
    before = k["p"].clone().contiguous()
    k["grad"][k["mask"]] = 1.0
    C.push(args, native.ptr(k["lsync"]), 0, native.current_stream())
    torch.cuda.synchronize()
    assert torch.equal(before, k["p"].contiguous()) and torch.all(k["grad"] == 0)
    assert int(k["ctrl"][5]) == 1 and int(k["ctrl"][3]) == 0


@pytest.mark.parametrize("lock_mode", [0, 1])
def test_pull_copies_publish_buffer(C, lock_mode):
    n16, n32 = 64 * 1000, 4 * 300
    src = torch.randn(n16, device="cuda").to(torch.bfloat16)
    dst = torch.zeros_like(src)
    sstate = torch.randn(n32, 4, device="cuda")
    s32 = sstate[:, 0].contiguous()
    d32 = torch.zeros_like(s32)
    ctrl = torch.zeros(C.CTRL_WORDS, dtype=torch.int32, device="cuda")
    ctrl[1] = 41
    seen = torch.zeros(1, dtype=torch.int32, device="cuda")
    lsync = torch.zeros(8, dtype=torch.int32, device="cuda")
    d = dict(src=native.ptr(src), dst=native.ptr(dst), src_state=native.ptr(sstate), dst_f32=native.ptr(d32),
             n_bf16=n16, n_f32=n32, ctrl=native.ptr(ctrl), seen_version=native.ptr(seen), lock_mode=lock_mode)
    for _ in range(2):
        C.pull(d, native.ptr(lsync), 0, native.current_stream())
    torch.cuda.synchronize()
    assert torch.equal(src, dst) and torch.equal(s32, d32) and int(seen[0]) == 41 and int(ctrl[0]) == 0


def test_device_rwlock_word(C):
    ctrl = torch.zeros(C.CTRL_WORDS, dtype=torch.int32, device="cuda")
    st = native.current_stream()
    C.lock_op(native.ptr(ctrl), 0, st); C.lock_op(native.ptr(ctrl), 0, st)
    torch.cuda.synchronize()
    assert int(ctrl[0]) == 2
    C.lock_op(native.ptr(ctrl), 1, st); C.lock_op(native.ptr(ctrl), 1, st)
    C.lock_op(native.ptr(ctrl), 2, st)
    torch.cuda.synchronize()
    assert int(ctrl[0]) == 1 << 16
    C.lock_op(native.ptr(ctrl), 3, st)
    torch.cuda.synchronize()
    assert int(ctrl[0]) == 0


def test_plan_capture_replay(C):
    x = torch.randn(64, 32, device="cuda")
    out = torch.zeros(64, 32, dtype=torch.bfloat16, device="cuda")
    plan = C.Plan()
    plan.add_cast_transpose(native.ptr(x), 32, 0, native.ptr(out), 32, 0, 0, 64, 32)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        plan.run(st.cuda_stream)
        st.synchronize()
        plan.capture(st.cuda_stream)
        out.zero_()
        plan.replay(st.cuda_stream)
    st.synchronize()
    assert torch.equal(out, x.to(torch.bfloat16))


def test_plan_branches_fork_join(C):
    x = torch.randn(64, 32, device="cuda")
    a = torch.zeros(64, 32, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros(64, 32, dtype=torch.bfloat16, device="cuda")
    plan = C.Plan()
    plan.fork(1)
    plan.branch(1)
    plan.add_cast_transpose(native.ptr(x), 32, 0, native.ptr(a), 32, 0, 0, 64, 32)
    plan.branch(0)
    plan.add_cast_transpose(native.ptr(x), 32, 0, native.ptr(b), 32, 0, 0, 64, 32)
    plan.join(1)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        plan.run(st.cuda_stream)
        st.synchronize()
        plan.capture(st.cuda_stream)
        a.zero_(); b.zero_()
        plan.replay(st.cuda_stream)
    st.synchronize()
    assert torch.equal(a, x.to(torch.bfloat16)) and torch.equal(b, x.to(torch.bfloat16))
    assert plan.graph_nodes() >= 2 and plan.names() == ["cast_transpose@1", "cast_transpose"]


def test_im2col_and_col2im(C):
    n, h, w, c, kh, kw = 5, 12, 12, 32, 3, 3
    x = torch.randn(n, h, w, c, device="cuda").to(torch.bfloat16)
    oh, ow = h - kh + 1, w - kw + 1
    M, K = n * oh * ow, kh * kw * c
    ldK, ldM = round_up(K, 8), round_up(M, 8)
    out = torch.zeros(M, ldK, dtype=torch.bfloat16, device="cuda")
    outT = torch.zeros(K, ldM, dtype=torch.bfloat16, device="cuda")
    st = native.current_stream()
    C.im2col(native.ptr(x), n, h, w, c, kh, kw, native.ptr(out), ldK, native.ptr(outT), ldM, st)
    torch.cuda.synchronize()
    ref = torch.nn.functional.unfold(x.float().permute(0, 3, 1, 2), (kh, kw))            # [n, c*kh*kw, L] in (c, kh, kw) order
    ref = ref.reshape(n, c, kh * kw, oh * ow).permute(0, 3, 2, 1).reshape(M, K)       # -> (kh, kw, c) order
    assert torch.equal(out[:, :K].float(), ref) and torch.equal(outT[:, :M].float().t(), ref)
    # col2im == adjoint of im2col
    dcols = torch.randn(M, ldK, device="cuda").to(torch.bfloat16)
    din = torch.zeros(n, h, w, c, dtype=torch.bfloat16, device="cuda")
    C.col2im(native.ptr(dcols), ldK, n, h, w, c, kh, kw, native.ptr(din), st)
    torch.cuda.synchronize()
    d = dcols[:, :K].float().reshape(n, oh * ow, kh * kw, c).permute(0, 3, 2, 1).reshape(n, c * kh * kw, oh * ow)
    ref_in = torch.nn.functional.fold(d, (h, w), (kh, kw)).permute(0, 2, 3, 1)
    torch.testing.assert_close(din.float(), ref_in, rtol=2e-2, atol=5e-2)


def test_maxpool_fwd_bwd(C):
    n, h, w, c = 4, 10, 10, 64
    a = torch.relu(torch.randn(n, h, w, c, device="cuda")).to(torch.bfloat16)
    oh, ow = h // 2, w // 2
    out = torch.zeros(n, oh, ow, c, dtype=torch.bfloat16, device="cuda")
    am = torch.zeros(n, oh, ow, c, dtype=torch.uint8, device="cuda")
    ldB = round_up(n, 8)
    outT = torch.zeros(oh * ow * c, ldB, dtype=torch.bfloat16, device="cuda")
    st = native.current_stream()
    C.maxpool_fwd(native.ptr(a), n, h, w, c, native.ptr(out), native.ptr(am), native.ptr(outT), ldB, st)
    torch.cuda.synchronize()
    af = a.float().permute(0, 3, 1, 2).requires_grad_(True)
    ref = torch.nn.functional.max_pool2d(torch.relu(af), 2)
    assert torch.equal(out.float(), ref.detach().permute(0, 2, 3, 1))
    assert torch.equal(outT[:, :n].float().t(), ref.detach().permute(0, 2, 3, 1).reshape(n, -1))
    dout = torch.randn(n, oh, ow, c, device="cuda").to(torch.bfloat16)
    ref.backward(dout.float().permute(0, 3, 1, 2))
    M = n * h * w
    ldM = round_up(M, 8)
    dz = torch.zeros(M, c, dtype=torch.bfloat16, device="cuda")
    dzT = torch.zeros(c, ldM, dtype=torch.bfloat16, device="cuda")
    db = torch.zeros(c, device="cuda")
    C.maxpool_bwd(native.ptr(dout), native.ptr(am), n, h, w, c, native.ptr(a), 1, native.ptr(dz), c, native.ptr(dzT), ldM, native.ptr(db), st)
    torch.cuda.synchronize()
    g = af.grad.permute(0, 2, 3, 1).reshape(M, c)
    # ties inside a window may pick a different (equal-valued) winner than torch: compare where unambiguous
    torch.testing.assert_close(dz.float().sum(), g.sum(), rtol=1e-2, atol=1e-1)
    mism = (dz.float() != g).float().mean().item()
    assert mism < 0.02, mism
    assert torch.equal(dzT[:, :M].float().t(), dz.float())
    torch.testing.assert_close(db, dz.float().sum(0), rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("n,h,w,cin,kh,kw,cout,act", [(5, 28, 28, 1, 5, 5, 32, "relu"), (3, 12, 12, 2, 3, 3, 16, "tanh"), (2, 9, 9, 3, 2, 2, 64, None)])
def test_conv_first_fused_fwd_and_wgrad(C, n, h, w, cin, kh, kw, cout, act):
    """First conv + bias + activation + 2x2 max-pool as one direct kernel, and its fused weight / bias gradient, against
    torch (conv2d -> act -> max_pool2d and autograd through them)."""
    import torch.nn.functional as F

    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(torch.bfloat16)
    K = kh * kw * cin
    wmat = (torch.randn(K, cout, device="cuda", generator=g) * 0.3).to(torch.bfloat16)      # [K = (dy, dx, ci), cout] (HWIO flattened)
    ld_w = round_up(K, 8)
    wT = torch.zeros(cout, ld_w, dtype=torch.bfloat16, device="cuda")
    wT[:, :K] = wmat.t()
    bias = torch.randn(cout, device="cuda", generator=g) * 0.1
    oh, ow = h - kh + 1, w - kw + 1
    ph, pw = oh // 2, ow // 2
    pooled = torch.zeros(n, ph, pw, cout, dtype=torch.bfloat16, device="cuda")
    argmax = torch.zeros(n, ph, pw, cout, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    C.conv_first_fwd(x.data_ptr(), n, h, w, cin, kh, kw, cout, wT.data_ptr(), ld_w, bias.data_ptr(), ACT[act], pooled.data_ptr(), argmax.data_ptr(), st)
    torch.cuda.synchronize()
    xt = x.float().permute(0, 3, 1, 2).requires_grad_(False)
    wt = wmat.float().reshape(kh, kw, cin, cout).permute(3, 2, 0, 1).clone().requires_grad_(True)
    bt = bias.clone().requires_grad_(True)
    conv = _act(F.conv2d(xt, wt, bt), act)
    ref = F.max_pool2d(conv, 2)[:, :, :ph, :pw]
    assert torch.allclose(pooled.float().permute(0, 3, 1, 2), ref, rtol=2e-2, atol=2e-2)
    # gradient of sum(g_pool * pooled) through the SAME arg-max positions the kernel recorded
    gp = torch.randn(n, ph, pw, cout, device="cuda", generator=g).to(torch.bfloat16)
    dW = torch.zeros(K, cout, device="cuda")
    db = torch.zeros(cout, device="cuda")
    C.conv_first_wgrad(x.data_ptr(), n, h, w, cin, kh, kw, cout, gp.data_ptr(), pooled.data_ptr(), argmax.data_ptr(), ACT[act], dW.data_ptr(),
                       db.data_ptr(), st)
    torch.cuda.synchronize()
    am = argmax.long().permute(0, 3, 1, 2)
    ys = 2 * torch.arange(ph, device="cuda").view(1, 1, ph, 1) + am // 2
    xs = 2 * torch.arange(pw, device="cuda").view(1, 1, 1, pw) + am % 2
    picked = conv[torch.arange(n, device="cuda").view(n, 1, 1, 1), torch.arange(cout, device="cuda").view(1, cout, 1, 1), ys, xs]
    # the kernel takes act'(.) from the bf16-rounded pooled value: use the same mask convention for ReLU ties
    (picked * gp.float().permute(0, 3, 1, 2)).sum().backward()
    ref_dW = wt.grad.permute(2, 3, 1, 0).reshape(K, cout)
    scale = max(1.0, ref_dW.abs().max().item())
    assert (dW - ref_dW).abs().max().item() < 3e-2 * scale
    assert torch.allclose(db, bt.grad, rtol=3e-2, atol=3e-2 * max(1.0, bt.grad.abs().max().item()))
