"""Dropout on conv and max-pool outputs on the GPU: the dropout twins of the pool kernels against the host Philox mask
(tests/dropout_ref.py) and float64, and the compiled training step of the zoo models ``dropout_cnn`` and
``conv_dropout_cnn`` against the image-dropout oracle of tests/test_conv_dropout.py, in every plan variant that applies,
with push in every push mode, in its forward-only plans and through a training session.
"""
import numpy as np
import pytest
import torch

import test_conv_dropout as cd
import test_step_gradients as sg
from sparkflow_b200.ops import native
from dropout_ref import dropout_mask, dropout_seed
from push_helpers import wait_pushes

pytestmark = pytest.mark.gpu

KEEPS = (0.5, 0.75, 0.9)
CTRS = (0, 1, 2 ** 32 - 1)
STREAMS = (0, 3, 0xFFFFFFFF)
# (kh, kw, sh, sw, padding): the 2x2 kernel, and the general kernel VALID, SAME and with overlapping windows
POOLS = [(2, 2, 2, 2, "fast"), (2, 2, 2, 2, "VALID"), (3, 3, 2, 2, "SAME"), (3, 3, 1, 1, "SAME"), (4, 3, 3, 2, "VALID")]
POOL_IDS = ["2x2", "gen2x2", "gen3x3s2same", "gen3x3s1same", "gen4x3valid"]
KEPT = 0x80


def _geom(H, W, kh, kw, sh, sw, pad):
    if pad == "SAME":
        oh, ow = -(-H // sh), -(-W // sw)
        return oh, ow, max((oh - 1) * sh + kh - H, 0) // 2, max((ow - 1) * sw + kw - W, 0) // 2
    return (H - kh) // sh + 1, (W - kw) // sw + 1, 0, 0


def _ctr_word(ctr):
    return torch.from_numpy(np.array([ctr], dtype=np.uint32).view(np.int32)).cuda()


def _pool_fwd(C, x, B, H, W, c, cfg, drop=None):
    """pooled output and argmax of the plain kernel, or of its dropout twin with drop = (keep, seed, stream, ctr word)"""
    kh, kw, sh, sw, pad = cfg
    oh, ow, pt, pl = _geom(H, W, kh, kw, sh, sw, "VALID" if pad == "fast" else pad)
    out = torch.full((B, oh * ow * c), 7.0, dtype=torch.bfloat16, device="cuda")
    am = torch.full((B, oh * ow * c), 0x55, dtype=torch.uint8, device="cuda")
    st = native.current_stream()
    P = native.ptr
    if pad == "fast":
        if drop:
            C.image_dropout.maxpool_drop_fwd(P(x), B, H, W, c, P(out), P(am), drop[0], drop[1], drop[2], P(drop[3]), st)
        else:
            C.maxpool_fwd(P(x), B, H, W, c, P(out), P(am), 0, 0, st)
    elif drop:
        C.image_dropout.maxpool_gen_drop_fwd(P(x), B, H, W, c, kh, kw, sh, sw, pt, pl, oh, ow, P(out), P(am), drop[0], drop[1], drop[2], P(drop[3]), st)
    else:
        C.maxpool_gen_fwd(P(x), B, H, W, c, kh, kw, sh, sw, pt, pl, oh, ow, P(out), P(am), st)
    torch.cuda.synchronize()
    return out, am, (oh, ow, pt, pl)


@pytest.mark.parametrize("cfg", POOLS, ids=POOL_IDS)
def test_pool_dropout_forward_matches_host_mask(cfg):
    """Small-integer inputs: the twin's output is the plain kernel's times mask / keep - bit for bit at keep 0.5, within
    one bf16 step otherwise - with the mask the host draws for the pooled matrix [B * OH * OW, C]; argmax bits 0-6 are
    the plain kernel's, bit 7 the mask.  Row counts cross 256-thread blocks; channel counts leave partial Philox groups."""
    C = native.cuda_ext()
    g = torch.Generator(device="cuda").manual_seed(5)
    k = 0
    for B, H, W, c in ((1, 6, 6, 8), (3, 9, 7, 12), (37, 12, 10, 24)):
        x = torch.randint(-8, 9, (B, H * W * c), device="cuda", generator=g).to(torch.bfloat16)
        ref_out, ref_am, (oh, ow, _, _) = _pool_fwd(C, x, B, H, W, c, cfg)
        for keep in KEEPS:
            for ctr in CTRS:
                stream, seed = STREAMS[k % 3], (0x9E3779B9 * (k + 1)) & 0xFFFFFFFF
                k += 1
                out, am, _ = _pool_fwd(C, x, B, H, W, c, cfg, (keep, seed, stream, _ctr_word(ctr)))
                tag = f"{cfg} B={B} {H}x{W}x{c} keep={keep} ctr={ctr} stream={stream}"
                m = torch.from_numpy(dropout_mask(B * oh * ow, c, np.float32(keep), seed, stream, ctr).reshape(B, -1)).cuda()
                assert torch.equal(am & 0x7F, ref_am), f"{tag}: winners differ from the plain kernel"
                assert torch.equal((am & KEPT) != 0, m), f"{tag}: argmax bit 7 is not the host mask"
                assert not bool((out[~m] != 0).any()), f"{tag}: a dropped element is non-zero"
                want = (ref_out.double() / keep).float().to(torch.bfloat16).double() * m
                got = out.double()
                if keep == 0.5:
                    assert torch.equal(got, want), f"{tag}: not bit-exact"
                else:
                    step = torch.ldexp(torch.ones_like(want), torch.frexp(want)[1] - 8)
                    assert bool(((got - want).abs() <= step).all()), f"{tag}: more than one bf16 step from pooled / keep"
                    assert float(m.double().mean()) == pytest.approx(keep, abs=0.25)


def _act64(z, act, alpha=0.1):
    f = {0: lambda t: t, 1: torch.relu, 2: torch.sigmoid, 3: torch.tanh, 4: torch.nn.functional.elu, 5: torch.selu,
         6: torch.nn.functional.softplus, 7: torch.nn.functional.softsign, 8: lambda t: torch.nn.functional.leaky_relu(t, alpha),
         9: torch.nn.functional.relu6}
    return f[act](z)


def _dact64(a, act, alpha=0.1):
    """act'(z) from a = act(z), as the kernels take it"""
    lam, al = 1.0507009873554805, 1.6732632423543772
    return {0: torch.ones_like(a), 1: (a > 0).double(), 2: a * (1 - a), 3: 1 - a * a, 4: torch.where(a > 0, 1.0, a + 1),
            5: torch.where(a > 0, lam, a + lam * al), 6: 1 - torch.exp(-a), 7: (1 - a.abs()) ** 2,
            8: torch.where(a > 0, 1.0, alpha), 9: ((a > 0) & (a < 6)).double()}[act]


def _act_arg(act, alpha=0.1):
    import struct
    return act | ((struct.unpack("<I", struct.pack("<f", alpha))[0] << 32) if act == 8 else 0)


@pytest.mark.parametrize("cfg", POOLS, ids=POOL_IDS)
def test_pool_dropout_backward_matches_float64(cfg):
    """The backward twins, every activation id: a dropout on the pooled output (g * mask / keep to the winner, the mask
    from argmax bit 7) and one on the conv output (act_out = act(z) * mask / keep, act' at act_out * keep, times
    1 / keep), in dz and the bias gradient, against float64 to within fp32 / one bf16 step."""
    C = native.cuda_ext()
    P = native.ptr
    gen = torch.Generator(device="cuda").manual_seed(9)
    B, H, W, c = 5, 11, 9, 40
    kh, kw, sh, sw, pad = cfg
    for act in range(10):
        for where in ("pool", "conv"):
            keep, seed, stream, ctr = 0.75, 0xABCDE + act, act, 3
            z = 1.5 * torch.randn(B, H, W, c, device="cuda", generator=gen, dtype=torch.float64)
            a = _act64(z, act)
            cm = torch.from_numpy(dropout_mask(B * H * W, c, np.float32(keep), seed, stream, ctr).reshape(B, H, W, c)).cuda()
            if where == "conv":
                a = a * cm / keep
            a_bf = a.float().to(torch.bfloat16)
            drop = (keep, seed, stream, _ctr_word(ctr)) if where == "pool" else None
            pooled, am, (oh, ow, pt, pl) = _pool_fwd(C, a_bf.reshape(B, -1), B, H, W, c, cfg, drop)
            dout = torch.randn(B, oh * ow * c, device="cuda", generator=gen).to(torch.bfloat16)
            dz = torch.full((B * H * W, c), 3.0, dtype=torch.bfloat16, device="cuda")
            db = torch.zeros(c, device="cuda")
            pk, ak = (keep, 0.0) if where == "pool" else (0.0, keep)
            st = native.current_stream()
            if pad == "fast":
                C.image_dropout.maxpool_drop_bwd(P(dout), P(am), B, H, W, c, P(a_bf), _act_arg(act), pk, ak, P(dz), c, P(db), st)
            else:
                C.image_dropout.maxpool_gen_drop_bwd(P(dout), P(am), B, H, W, c, kh, kw, sh, sw, pt, pl, oh, ow, P(a_bf), _act_arg(act), pk, ak, P(dz), c,
                                       P(db), st)
            torch.cuda.synchronize()
            # float64: route every pooled gradient to its winner
            win = (am & 0x7F).long().reshape(B, oh, ow, c)
            g = dout.double().reshape(B, oh, ow, c)
            if where == "pool":
                g = g * ((am & KEPT) != 0).reshape(B, oh, ow, c).double() / keep
            oy = torch.arange(oh, device="cuda").view(1, oh, 1, 1) * sh - pt + win // kw
            ox = torch.arange(ow, device="cuda").view(1, 1, ow, 1) * sw - pl + win % kw
            flat = (oy * W + ox).reshape(B, oh * ow, c)
            gin = torch.zeros(B, H * W, c, dtype=torch.float64, device="cuda").scatter_add_(1, flat, g.reshape(B, oh * ow, c))
            a_st = a_bf.double().reshape(B, H * W, c)
            if where == "conv":
                d = torch.where(a_st != 0, _dact64(a_st * keep, act) / keep, torch.zeros_like(a_st))
                if act == 9:
                    sat = float(torch.tensor(6.0 / keep).float().to(torch.bfloat16))
                    d = ((a_st > 0) & (a_st < sat)).double() / keep
            else:
                d = _dact64(a_st, act)
            ref = (gin * d).reshape(B * H * W, c)
            got = dz.double()
            tag = f"{cfg} act={act} dropout on the {where} output"
            tol = torch.ldexp(torch.ones_like(ref), torch.frexp(ref)[1] - 8) + 1e-5 * gin.abs().reshape(B * H * W, c).max()
            assert bool(((got - ref).abs() <= tol).all()), f"{tag}: dz max err {float((got - ref).abs().max()):.3e}"
            assert torch.allclose(db.double(), ref.sum(0), rtol=1e-4, atol=1e-4 * float(ref.abs().sum(0).max())), tag


def test_act_dropout_backward_matches_float64():
    """act_drop_bwd_bias: dz = g * mask / keep * act'(a * keep) from the stored a = act(z) * mask / keep, every activation"""
    C = native.cuda_ext()
    P = native.ptr
    gen = torch.Generator(device="cuda").manual_seed(11)
    for M, c in ((1, 8), (77, 40), (1000, 64)):
        for act in range(10):
            keep = KEEPS[act % 3]
            m = torch.from_numpy(dropout_mask(M, c, np.float32(keep), 77, act, 5)).cuda()
            a_bf = (_act64(1.5 * torch.randn(M, c, device="cuda", generator=gen, dtype=torch.float64), act) * m / keep).float().to(torch.bfloat16)
            g = torch.randn(M, c, device="cuda", generator=gen).to(torch.bfloat16)
            dz = torch.zeros(M, c, dtype=torch.bfloat16, device="cuda")
            db = torch.zeros(c, device="cuda")
            C.image_dropout.act_drop_bwd_bias(P(g), c, M, c, P(a_bf), _act_arg(act), keep, P(dz), c, P(db), native.current_stream())
            torch.cuda.synchronize()
            a = a_bf.double()
            d = torch.where(a != 0, _dact64(a * keep, act) / keep, torch.zeros_like(a))
            if act == 9:
                d = ((a > 0) & (a < float(torch.tensor(6.0 / keep).float().to(torch.bfloat16)))).double() / keep
            ref = g.double() * d
            tol = torch.ldexp(torch.ones_like(ref), torch.frexp(ref)[1] - 8) + 1e-6
            assert bool(((dz.double() - ref).abs() <= tol).all()), (M, c, act)
            assert torch.allclose(db.double(), ref.sum(0), rtol=1e-4, atol=1e-4), (M, c, act)


# ----------------------------------------------------------------------------------------------------------------------
# the compiled training step
# ----------------------------------------------------------------------------------------------------------------------
def _register(name):
    """make the zoo model known to test_step_gradients' worker and step helpers"""
    ir, lp = cd.model(name)
    sg._MODEL_CACHE[name] = (ir, lp, "y:0")
    return ir, lp


VARIANTS = dict(sg.VARIANTS, pair={"SPARKFLOW_GEMM_PAIR": "1"})
STEP_CASES = [(n, v) for n in cd.NAMES for v in ("default", "unfused_loss", "lowered_conv1", "no_branches", "pair")]


def _image_drop_layers(lp):
    return [i for i, l in enumerate(lp.layers) if l.dropout_keep and l.kind in ("conv", "pool")]


def _masks_of_step(tag, lp, dbg, B, worker_index=0, ctr=None):
    """host masks of every dropout layer at the counter the step read, after checking the recorded parameters"""
    seeds, word = set(), None
    for i, l in enumerate(lp.layers):
        if l.dropout_keep:
            r = dbg[i]["drop"]
            assert r["keep"] == l.dropout_keep and r["stream"] == i, (tag, i, r)
            assert r["seed"] == dropout_seed(worker_index, native.ptr(r["ctr"])), f"{tag}: layer {i} seed"
            seeds.add(r["seed"])
            word = r["ctr"]
    assert len(seeds) == 1, tag
    if ctr is None:
        ctr = int(word.cpu().view(-1)[0]) & 0xFFFFFFFF
    return cd.host_masks(lp, B, seeds.pop(), ctr), ctr


def _check_stored(tag, lp, dbg, masks, B):
    """every stored image-dropout output is zero where the host mask drops; a pool's argmax bit 7 is the mask"""
    for i in _image_drop_layers(lp):
        l = lp.layers[i]
        m = torch.from_numpy(masks[i])
        if l.kind == "conv":
            a = dbg[i]["act_out"].cpu().reshape(m.shape)
        else:
            a = dbg[i]["pooled"].cpu().reshape(m.shape)
            assert torch.equal((dbg[i]["argmax"].cpu().reshape(m.shape) & KEPT) != 0, m), f"{tag}: layer {i} argmax bit 7"
        assert not bool(((~m) & (a != 0)).any()), f"{tag}: layer {i}: units the host mask drops are non-zero"
        if l.act in ("Tanh", "Sigmoid"):
            # a kept tanh / sigmoid unit is non-zero, but for the epilogue's tanh of |z| below ~3e-8, which rounds to 0
            # (its 1 - exp(-2|z|)): allow one in 10^5
            zero = int((m & (a == 0)).sum())
            assert zero <= 1e-5 * m.numel(), f"{tag}: layer {i}: {zero} kept units are zero"


def _recorded(lp, dbg, B):
    argmax, relu = {}, {}
    dense = [i for i, l in enumerate(lp.layers) if l.kind == "dense"]
    for i, l in enumerate(lp.layers):
        if l.kind == "pool":
            argmax[i] = (dbg[i]["argmax"] & 0x7F).to(sg.DEV).long().reshape(B, *l.out_shape)
        if l.act == "Relu":
            if l.kind == "conv":
                relu[i] = dbg[i]["act_out"].to(sg.DEV).reshape(B, *l.out_shape) > 0
            elif i != dense[-1]:
                relu[i] = dbg[min(j for j in dense if j > i)]["a_in"][:, :l.out_shape[0]].to(sg.DEV) > 0
    return argmax, relu


def _compare(tag, name, lp, w, X, Y, got, loss, dbg, masks):
    B = X.shape[0]
    argmax, relu = _recorded(lp, dbg, B)
    l_ref, grads = cd.oracle(lp, w, X, Y, True, masks, argmax=argmax, relu_mask=relu)
    l_err = abs(loss - l_ref) / max(abs(l_ref), 1e-30)
    assert l_err <= cd.LOSS_TOL, f"{tag}: loss {loss} vs {l_ref}"
    fro, mx = sg._assert_grads(tag, lp.var_order, got, grads, cd.TOL[name])
    return fro, mx, l_err


def _kernels(names):
    return [n.split("@")[0] for n in names]


@pytest.mark.parametrize("name,variant", STEP_CASES)
def test_image_dropout_step_matches_oracle(name, variant, monkeypatch):
    """One step without push, staged and in-graph feeds: the stored conv / pool outputs against the host masks at the
    counter the step read (0), every gradient and the loss against the oracle with those masks."""
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    _, lp = _register(name)
    w = cd.weights(name)
    master, worker = sg._worker(name, w)
    worst = [0.0, 0.0, 0.0]
    pair = False
    try:
        for B in (1, 7, 130, 300):
            X, Y = cd.data(name, B, seed=B + 60)
            for feed in ("staged", "in_graph"):
                tag = f"{name}/{variant} B={B} {feed}"
                got, loss, dbg, names = sg._run_step(worker, B, X, Y, feed)
                assert "conv_first_fwd" not in _kernels(names), tag
                masks, ctr = _masks_of_step(tag, lp, dbg, B)
                assert ctr == 0, tag
                _check_stored(tag, lp, dbg, masks, B)
                worst = [max(a, b) for a, b in zip(worst, _compare(tag, name, lp, w, X, Y, got, loss, dbg, masks))]
                pair |= any(getattr(g, "pair", 0) == 1 for grp in worker._keep[-1] if isinstance(grp, list) for g in grp)
    finally:
        master.close()
    if variant != "pair":
        assert not pair
    print(f"[conv-dropout] {name}/{variant}: worst rel-Frobenius {worst[0]:.2e}, max-abs {worst[1]:.2e}, loss {worst[2]:.2e} "
          f"(tolerance {cd.TOL[name]}, {cd.LOSS_TOL})")


def _no_dropout_cnn():
    from sparkflow_b200.graph import tfcompat as tf
    x = tf.placeholder(tf.float32, shape=[None, 784], name="x")
    y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
    img = tf.reshape(x, shape=[-1, 28, 28, 1])
    c2 = tf.layers.conv2d(tf.layers.conv2d(img, 32, 3, activation=tf.nn.relu), 64, 3, activation=tf.nn.relu)
    h = tf.layers.dense(tf.layers.flatten(tf.layers.max_pooling2d(c2, 2, 2)), 128, activation=tf.nn.relu)
    logits = tf.layers.dense(h, 10)
    tf.argmax(logits, 1, name="out")
    return tf.losses.softmax_cross_entropy(y, logits)


def test_image_dropout_adds_no_pass():
    """dropout_cnn's step runs the kernels of the same graph without dropouts, the pool and its backward replaced by
    their dropout twins: the masks cost no pass of their own"""
    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.graph_utils import build_graph
    from sparkflow_b200.models.compiler import compile_graph

    ir0 = GraphIR.from_metagraph(build_graph(_no_dropout_cnn))
    sg._MODEL_CACHE["no_dropout_cnn"] = (ir0, compile_graph(ir0, "x:0", "y:0"), "y:0")
    _register("dropout_cnn")
    lists = {}
    for name in ("dropout_cnn", "no_dropout_cnn"):
        w = cd.weights("dropout_cnn")
        master, worker = sg._worker(name, w)
        try:
            X, Y = cd.data("dropout_cnn", 130, seed=1)
            lists[name] = _kernels(sg._run_step(worker, 130, X, Y, "staged")[3])
        finally:
            master.close()
    twin = {"maxpool_fwd": "maxpool_drop_fwd", "maxpool_bwd": "maxpool_drop_bwd"}
    assert lists["dropout_cnn"] == [twin.get(n, n) for n in lists["no_dropout_cnn"]], lists


PUSH_MODES = {"direct": {}, "served": dict(push="served"), "sharded2": dict(push="sharded", shards=2)}


@pytest.mark.parametrize("mode", list(PUSH_MODES))
def test_pushed_image_dropout_steps_advance_the_mask(mode):
    """Three steps with push: each reads the counter its predecessor's push left, stores the host masks at that
    counter (different from the previous step's) and delivers the oracle's gradient (momentum with learning rate 0
    leaves slot 0 equal to it)."""
    from sparkflow_b200.ops.optimizers import OptimizerSpec

    name, B, steps = "conv_dropout_cnn", 130, 3
    _, lp = _register(name)
    w = cd.weights(name)
    X, Y = cd.data(name, steps * B, seed=77)
    spec = OptimizerSpec.from_tf_kwargs("momentum", dict(learning_rate=0.0, momentum=0.0))
    master, worker = sg._worker(name, w, spec, **PUSH_MODES[mode])
    try:
        plan, bufs = worker.build_plan(B, 0, with_pull=True, with_push=True)
        dbg = worker.last_debug
        prev = None
        for k in range(steps):
            rows = slice(k * B, (k + 1) * B)
            tag = f"{name}/{mode} step {k}"
            masks, ctr = _masks_of_step(tag, lp, dbg, B)
            assert ctr == k, tag
            with torch.cuda.stream(worker.stream):
                bufs.x_stage.copy_(torch.from_numpy(X[rows]))
                bufs.y_stage.copy_(torch.from_numpy(Y[rows]))
            worker.run_plan(plan)
            worker.drain()
            assert wait_pushes(master, k + 1) == k + 1
            _check_stored(tag, lp, dbg, masks, B)
            if prev is not None:
                assert all(not np.array_equal(masks[i], prev[i]) for i in masks), f"{tag}: the previous step's mask"
            prev = masks
            _compare(tag, name, lp, w, X[rows], Y[rows], master.slot_arrays()[0], float(bufs.loss_out[0]), dbg, masks)
    finally:
        master.close()


@pytest.mark.parametrize("name", cd.NAMES)
def test_image_dropout_forward_plans_match_oracle(name):
    """predict and the forward + loss plan draw the masks of counter 0 under the seed without a counter address"""
    _, lp = _register(name)
    w = cd.weights(name)
    B = 130
    X, Y = cd.data(name, B, seed=41)
    masks = cd.host_masks(lp, B, dropout_seed(0), 0)
    with torch.no_grad():
        l_ref, out_ref = cd.forward(lp, w, X, Y, True, drop_mask=masks)[:2]
        other = cd.forward(lp, w, X, Y, True, drop_mask=cd.host_masks(lp, B, dropout_seed(0), 1))[1]
    master, worker = sg._worker(name, w)
    try:
        out = worker.predict(X, upto=None, post=None)
        fro, mx = sg._errors(out, out_ref.cpu().numpy())
        assert fro <= sg.FWD_TOL[0] and mx <= sg.FWD_TOL[1], (fro, mx)
        assert sg._errors(out, other.cpu().numpy())[0] > 0.05, "the output does not depend on the mask"
        plan, bufs = worker.build_forward_plan(B, with_loss=True, with_pull=True)
        with torch.cuda.stream(worker.stream):
            bufs.x_stage.copy_(torch.from_numpy(X))
            bufs.y_stage.copy_(torch.from_numpy(Y))
            bufs.loss_out.zero_()
            plan.run(worker.stream.cuda_stream)
        worker.stream.synchronize()
        loss = float(bufs.loss_out[0])
        assert abs(loss - float(l_ref)) <= cd.LOSS_TOL * abs(float(l_ref)), (loss, float(l_ref))
        print(f"[conv-dropout] {name} forward: rel-Frobenius {fro:.2e}, max-abs {mx:.2e}")
    finally:
        master.close()


@pytest.mark.parametrize("name", cd.NAMES)
def test_session_trains_image_dropout_natively(name, monkeypatch, capfd):
    """The session runs both models natively (the interpreter is patched to fail); a short run of dropout_cnn lowers the
    loss"""
    from sparkflow_b200.graph.executor import GraphProgram
    from sparkflow_b200.models import zoo
    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.parallel.session import TrainingSession

    def refuse(*a, **k):
        raise AssertionError("the interpreter ran")

    monkeypatch.setattr(GraphProgram, "forward", refuse)
    rng = np.random.default_rng(3)
    centers = rng.random((10, 784), dtype=np.float32)
    lab = rng.integers(0, 10, 1200)
    X = np.clip(centers[lab] + 0.2 * rng.normal(0, 1, (1200, 784)), 0, 1).astype(np.float32)
    Y = np.eye(10, dtype=np.float32)[lab]
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    sess = TrainingSession(zoo.build(name), "x:0", "y:0", spec, seed=0, devices=[0]).open()
    try:
        assert sess.engine_kind == "b200"
        eng = sess.make_engine(torch.device("cuda", 0))
        eng.load_partition(X, Y)
        l0 = eng.partition_loss()
        for k in range(12):
            eng.train(slice((k % 4) * 300, (k % 4) * 300 + 300), pull=True)
        eng.finish()
        l1 = eng.partition_loss()
        assert np.isfinite(l1) and (name != "dropout_cnn" or l1 < 0.7 * l0), (l0, l1)
        assert sess.counters()["pushes"] == 12
    finally:
        sess.close()
    assert "engine=torch" not in capfd.readouterr().err
