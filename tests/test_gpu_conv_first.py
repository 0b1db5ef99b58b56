"""The fused first convolution (csrc/conv.cu: conv_first_fwd_kernel, conv_first_wgrad_kernel) against the float64
reference of tests/conv_ref.py, at every kernel instance and shared-memory path, at one image, a few, and more images than
the grids have CTAs; the planner's admission rule against both launchers; and a first conv past the weight gradient's
budget trained through the lowered path.

With integer operands (none and ReLU) the forward and the weight gradient are exact in fp32 whatever order the atomics
land in, so they must be bit-equal to float64; real-valued operands and sigmoid / tanh are held to the element-wise
bounds conv_ref derives from the kernels' arithmetic (test_bounds_reject_plausible_faults shows those bounds can fail).
The reference self-tests need no GPU; every GPU test carries its own mark."""
import pytest
import torch

import conv_ref as R
from sparkflow_b200.ops import native
from sparkflow_b200.parallel.plan_builder import fused_first_conv

# (h, w, cin, k, padding, cout): what each pins is asserted by test_cases_cover_every_launch_path
GEOMS = {
    "cnn": (28, 28, 1, 5, "VALID", 32),             # <5,5,1>, staged wgrad above the 48 KiB default (52,800 B)
    "cnn_same": (28, 28, 1, 5, "SAME", 32),         # SAME border, 62,080 B
    "k3c1_cout8": (28, 28, 1, 3, "VALID", 8),       # <3,3,1>, cout = 8: 32 groups per channel
    "cifar": (32, 32, 3, 3, "SAME", 64),            # <3,3,3>, unstaged wgrad
    "odd29": (31, 31, 3, 3, "VALID", 16),           # odd conv output: its last row and column are never pooled
    "big_fwd": (64, 64, 3, 3, "SAME", 8),           # forward at 52,272 B (opt-in), unstaged wgrad
    "k64_valid": (20, 20, 4, 4, "VALID", 16),       # <0,0,0> at K = 64
    "k64_same": (20, 20, 4, 4, "SAME", 16),         # even kernel under SAME: 1 pad in front, 2 behind
    "k49": (27, 27, 1, 7, "SAME", 64),              # K = 49, unstaged
    "tiny": (9, 9, 2, 3, "VALID", 8),               # odd output (7)
    "wgrad_cap": (62, 62, 3, 4, "VALID", 8),        # wgrad at 96,304 B, just under the cap
}
ALL_ACTS = ("cnn", "k3c1_cout8", "cifar", "k64_same")   # one geometry per template instance, one runtime-shape one
BATCHES = ("1", "7", "large")


def _cases():
    out = []
    for g in GEOMS:
        for b in BATCHES:
            out.append((g, b, "relu", True))
            if g in ALL_ACTS:
                out += [(g, b, a, True) for a in (None, "sigmoid", "tanh")]
                out += [(g, b, a, False) for a in ("sigmoid", "tanh")]
            if g in ("cnn", "k49", "wgrad_cap") and b != "1":
                out.append((g, b, "relu", False))
    return out


CASES = _cases()


def _geometry(h, w, k, padding):
    """(oh, ow, pad_top, pad_left)"""
    if padding == "SAME":
        return h, w, R.same_pads(k)[0], R.same_pads(k)[0]
    return h - k + 1, w - k + 1, 0, 0


def _batch(b):
    return {"1": 1, "7": 7, "large": 4 * native.num_sms() + 5}[b]


@pytest.fixture(scope="module")
def C():
    return native.cuda_ext()


# ------------------------------------------------------------------------------------------------------------------
# without a GPU: the case table and the bounds
# ------------------------------------------------------------------------------------------------------------------
def test_cases_cover_every_launch_path():
    """Which instance, staging path and grid a launch takes is not observable from outside; computed with the launchers'
    formulas (conv_first_fwd_launch / conv_first_wgrad_launch in csrc/conv.cu), the cases reach every one of them."""
    sms = native.num_sms()
    seen = set()
    for name, (h, w, cin, k, padding, cout) in GEOMS.items():
        oh, ow, pt, pl = _geometry(h, w, k, padding)
        K = k * k * cin
        fwd = R.fwd_smem(k, k, cin, cout, oh, ow)
        wg, staged = R.wgrad_smem(k, k, cin, cout, oh, ow)
        assert wg <= R.MAX_SMEM and fwd <= R.MAX_SMEM, name
        seen |= {("instance", R.instance(k, k, cin)), ("staged", staged), ("K", K), ("cout", cout)}
        seen |= {("fwd opt-in", fwd > 48 * 1024), ("wgrad opt-in", wg > 48 * 1024), ("odd output", oh % 2 == 1)}
        if padding == "SAME" and k % 2 == 0:
            seen.add(("even SAME", (pt, k - 1 - pt)))
        if wg > R.MAX_SMEM - 2048:
            seen.add(("wgrad at the cap", True))
        n = _batch("large")
        parts, grid = R.fwd_parts(n, cout, oh, ow, sms)
        assert n * parts > grid, f"{name}: the forward's CTAs must loop over several (image, part) items"
        assert n > R.wgrad_grid(n, sms), f"{name}: the weight gradient must have more images than CTAs"
        seen.add(("large-batch parts", min(parts, 2)))
    for want in [("instance", (5, 5, 1)), ("instance", (3, 3, 1)), ("instance", (3, 3, 3)), ("instance", (0, 0, 0)),
                 ("staged", True), ("staged", False), ("K", 49), ("K", 64), ("cout", 8), ("fwd opt-in", True),
                 ("wgrad opt-in", True), ("odd output", True), ("even SAME", (1, 2)), ("wgrad at the cap", True),
                 ("large-batch parts", 1), ("large-batch parts", 2)]:
        assert want in seen, want
    assert {R.instance(GEOMS[g][3], GEOMS[g][3], GEOMS[g][2]) for g in ALL_ACTS} == {(5, 5, 1), (3, 3, 1), (3, 3, 3), (0, 0, 0)}


def _fault_setup(act):
    """a small real-valued case on the CPU: (xp, gz, argmax, dW0, db0, reference dW / db and their bounds, dims)"""
    n, h, cin, k, cout = 3, 12, 2, 3, 16
    oh = ow = h - k + 1
    ph, pw = oh // 2, ow // 2
    x, wT, bias = R.operands(n, h, h, cin, k, k, cout, False, 11, "cpu")
    xp = R.pad_image(x, k, k, 0, 0, oh, ow)
    a, _ = R.forward(xp, R.filters(wT, k, k, cin), bias, k, k, oh, ow, act)
    best, am = R.pool(a, ph, pw)
    pooled = best.float().to(torch.bfloat16)
    g = R.pool_grad(n, ph, pw, cout, False, 11, "cpu").double()
    gz = g * R.dact64(pooled, act)
    dW0 = torch.randint(-5, 6, (k * k * cin, cout), generator=torch.Generator().manual_seed(5)).float()
    db0 = torch.randint(-5, 6, (cout,), generator=torch.Generator().manual_seed(6)).float()
    dW, db, T = R.wgrad(xp, gz, am, k, k)
    eW, eb = R.wgrad_bound(gz, T, dW0, db0, n, cout, oh, ow, native.num_sms())
    return dict(xp=xp, g=g, gz=gz, am=am, k=k, cout=cout, n=n, ph=ph, pw=pw, dW0=dW0.double(), db0=db0.double(),
                dW=dW0.double() + dW, db=db0.double() + db, eW=eW, eb=eb)


def _faults(s):
    """(what, dW, db) of the weight gradient computed with one plausible fault"""
    k, xp, gz, am = s["k"], s["xp"], s["gz"], s["am"]
    taps = [(ty, tx) for ty in range(k) for tx in range(k)]

    def run(gz_=gz, **kw):
        dW, db, _ = R.wgrad(xp, gz_, am, k, k, **kw)
        return s["dW0"] + dW, s["db0"] + db

    no_last = gz.clone()
    no_last[-1] = 0
    lost = gz.clone().reshape(s["n"], -1, s["cout"])
    lost[0, ::R.THREADS // s["cout"]] = 0                        # group 0 of the first CTA: pixels 0, n_grp, 2 n_grp, ...
    yield ("a tap shifted by one column", *run(taps=[(0, 1)] + taps[1:]))
    yield ("dy and dx swapped", *run(taps=[(tx, ty) for ty, tx in taps]))
    yield ("the window origin instead of the winner", *run(origin=True))
    yield ("the last image dropped", *run(no_last))
    yield ("act' omitted", *run(s["g"]))
    yield ("one group's partial sum lost", *run(lost.reshape(gz.shape)))


@pytest.mark.parametrize("act", ["relu", "sigmoid", "tanh"])
def test_bounds_reject_plausible_faults(act):
    """The real-valued weight-gradient comparison can fail: fp32 roundings of the reference pass its bound, and each
    fault is rejected in dW or db."""
    s = _fault_setup(act)
    assert R.fraction(s["dW"].float(), s["dW"], s["eW"]) <= 1.0
    assert R.fraction(s["db"].float(), s["db"], s["eb"]) <= 1.0
    for what, dW, db in _faults(s):
        frac = max(R.fraction(dW, s["dW"], s["eW"]), R.fraction(db, s["db"], s["eb"]))
        print(f"[conv-first] {act} with {what}: {frac:.1f} x the bound")
        assert frac > 1.0, f"{act}: the bound accepts the weight gradient with {what}"


def test_forward_bound_rejects_a_wrong_winner():
    """the real-valued forward check refuses the second-best winner of a window and a pooled value one bf16 step off"""
    n, h, cin, k, cout = 2, 10, 1, 3, 8
    oh = ow = h - k + 1
    x, wT, bias = R.operands(n, h, h, cin, k, k, cout, False, 3, "cpu")
    a, e = R.forward(R.pad_image(x, k, k, 0, 0, oh, ow), R.filters(wT, k, k, cin), bias, k, k, oh, ow, "tanh")
    best, am = R.pool(a, oh // 2, ow // 2)
    pooled = best.float().to(torch.bfloat16)
    R.check_forward("clean", a, e, pooled, am.to(torch.uint8), False)
    second = R.windows(a, oh // 2, ow // 2).argsort(-1, descending=True)[..., 1]
    with pytest.raises(AssertionError, match="below their window maximum"):
        R.check_forward("second", a, e, pooled, second.to(torch.uint8), False)
    off = (pooled.float() * (1 + 2.0 ** -5)).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="pooled value"):
        R.check_forward("off", a, e, off, am.to(torch.uint8), False)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernels against float64
# ------------------------------------------------------------------------------------------------------------------
GUARD = 1000


def _launch(C, g, n, act, exact, seed, nulls=False):
    """Both launches into sentinel-filled buffers with a guard region past them.  Returns the operands and the outputs."""
    h, w, cin, k, padding, cout = GEOMS[g]
    oh, ow, pt, pl = _geometry(h, w, k, padding)
    ph, pw = oh // 2, ow // 2
    K = k * k * cin
    dev = torch.device("cuda")
    lim = 3 if act == "relu" else 1                   # {-1, 0, 1}: ties among the none / sigmoid / tanh maxima too
    x, wT, bias = R.operands(n, h, w, cin, k, k, cout, exact, seed, dev, lim)
    if nulls:
        bias = None
    total = n * ph * pw * cout
    pooled_buf = torch.full((total + GUARD,), float("nan"), dtype=torch.bfloat16, device=dev)
    am_buf = torch.full((total + GUARD,), 0xEE, dtype=torch.uint8, device=dev)
    st = native.current_stream()
    geo = dict(pad_top=pt, pad_left=pl, out_h=oh, out_w=ow)
    C.conv_first_fwd(native.ptr(x), n, h, w, cin, k, k, cout, native.ptr(wT), wT.shape[1], native.ptr(bias), R.ACT[act],
                     native.ptr(pooled_buf), native.ptr(am_buf), st, **geo)
    gp = R.pool_grad(n, ph, pw, cout, exact, seed, dev, lim)
    gen = torch.Generator().manual_seed(seed + 2)
    dW0 = torch.randint(-50, 51, (K * cout,), generator=gen).float().to(dev)
    db0 = torch.randint(-50, 51, (cout,), generator=gen).float().to(dev)
    dW_buf = torch.full((K * cout + GUARD,), 1234.5, device=dev)
    db_buf = torch.full((cout + GUARD,), 1234.5, device=dev)
    dW_buf[:K * cout], db_buf[:cout] = dW0, db0
    C.conv_first_wgrad(native.ptr(x), n, h, w, cin, k, k, cout, native.ptr(gp), native.ptr(pooled_buf), native.ptr(am_buf),
                       R.ACT[act], native.ptr(dW_buf), 0 if nulls else native.ptr(db_buf), st, **geo)
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    return dict(x=x, wT=wT, bias=bias, gp=gp, dW0=dW0.view(K, cout), db0=db0, pooled_buf=pooled_buf, am_buf=am_buf,
                dW_buf=dW_buf, db_buf=db_buf, geo=(h, w, cin, k, cout, oh, ow, pt, pl, ph, pw, K, total))


def _check(C, g, n, act, exact, seed, nulls=False):
    r = _launch(C, g, n, act, exact, seed, nulls)
    h, w, cin, k, cout, oh, ow, pt, pl, ph, pw, K, total = r["geo"]
    tag = f"{g} n={n} {act} {'exact' if exact else 'real'}{' null bias / db' if nulls else ''}"
    # layout: every pooled word and argmax byte written, nothing past them
    pooled, am = r["pooled_buf"][:total].view(n, ph, pw, cout), r["am_buf"][:total].view(n, ph, pw, cout)
    assert not bool(pooled.isnan().any()), f"{tag}: pooled outputs left unwritten"
    assert bool(r["pooled_buf"][total:].isnan().all()) and bool((r["am_buf"][total:] == 0xEE).all()), f"{tag}: wrote past the pooled output"
    assert bool((r["dW_buf"][K * cout:] == 1234.5).all()) and bool((r["db_buf"][cout:] == 1234.5).all()), f"{tag}: wrote past dW / db"
    if nulls:
        assert torch.equal(r["db_buf"][:cout], r["db0"]), f"{tag}: db written with a null db"
    # forward
    xp = R.pad_image(r["x"], k, k, pt, pl, oh, ow)
    a, e = R.forward(xp, R.filters(r["wT"], k, k, cin), r["bias"], k, k, oh, ow, act)
    ties = R.check_forward(tag, a, e, pooled, am, exact and act in (None, "relu"))
    if exact:
        R.check_tie_rule(tag, a, am)
        assert ties > 0, f"{tag}: no tied window, the tie rule went unexercised"
    # weight and bias gradient at the kernel's recorded winners, act' at its stored pooled value
    gz = r["gp"].double() * R.dact64(pooled, act)
    dW, db, T = R.wgrad(xp, gz, am, k, k)
    dW, db = r["dW0"].double() + dW, r["db0"].double() + db
    got_dW, got_db = r["dW_buf"][:K * cout].view(K, cout), r["db_buf"][:cout]
    if exact and act in (None, "relu"):
        assert float((T + r["dW0"].double().abs()).max()) < 2 ** 24      # every partial sum is an fp32 integer
        assert torch.equal(got_dW.double(), dW), f"{tag}: dW differs from float64 at {int((got_dW.double() != dW).sum())} words"
        if not nulls:
            assert torch.equal(got_db.double(), db), f"{tag}: db differs from float64"
    else:
        eW, eb = R.wgrad_bound(gz, T, r["dW0"], r["db0"], n, cout, oh, ow, native.num_sms())
        frac = R.fraction(got_dW, dW, eW)
        assert frac <= 1.0, f"{tag}: dW off by {frac:.2f} x its bound"
        if not nulls:
            frac = R.fraction(got_db, db, eb)
            assert frac <= 1.0, f"{tag}: db off by {frac:.2f} x its bound"


@pytest.mark.gpu
@pytest.mark.parametrize("geom,batch,act,exact", CASES)
def test_conv_first_matches_float64(C, geom, batch, act, exact):
    """Forward (pooled value and winner) and weight / bias gradient (accumulated onto non-zero start values) against
    float64; n = 7 with integer ReLU operands passes a null bias and a null db."""
    n = _batch(batch)
    _check(C, geom, n, act, exact, seed=CASES.index((geom, batch, act, exact)), nulls=exact and act == "relu" and batch == "7")


# ------------------------------------------------------------------------------------------------------------------
# GPU: the planner against the launchers
# ------------------------------------------------------------------------------------------------------------------
def _sweep():
    """(cin, k, cout, padding, image sizes): around the largest square image that fits both the 64 KiB image rule and
    the weight gradient's 96 KiB"""
    out = []
    for cin in (1, 2, 3, 4):
        for k in range(3, 9):
            if k * k * cin > 64:
                continue
            for cout in (8, 16, 32, 64):
                for padding in ("VALID", "SAME"):
                    def fits(s):
                        oh = s - k + 1 if padding == "VALID" else s
                        hp = oh + k - 1
                        return hp * hp * cin * 4 <= 64 * 1024 and R.wgrad_smem(k, k, cin, cout, oh, oh)[0] <= R.MAX_SMEM
                    s = k + 1
                    while fits(s + 1):
                        s += 1
                    out.append((cin, k, cout, padding, (s - 1, s, s + 1, s + 2)))
    return out


@pytest.mark.gpu
def test_planner_admits_only_what_both_launchers_accept(C):
    """Every first conv the planner admits runs through both direct launches; every one past the weight gradient's
    shared-memory budget is refused by the planner (and by the launcher, on the host: rc -8 before anything is
    enqueued).  The 64 KiB image rule still refuses some shapes the launchers would take."""
    dev = torch.device("cuda")
    st = native.current_stream()
    admitted = refused_by_budget = 0
    for cin, k, cout, padding, sizes in _sweep():
        for s in sizes:
            lp = R.first_conv_plan(s, s, cin, k, cout, padding.lower())[1]
            oh = lp.layers[1].out_shape[0]
            pt = lp.layers[1].pads[0]
            over = R.wgrad_smem(k, k, cin, cout, oh, oh)[0] > R.MAX_SMEM
            ok = fused_first_conv(lp) is not None
            tag = f"{s}x{s}x{cin} k={k} cout={cout} {padding}"
            assert not (ok and over), f"{tag}: admitted past the weight gradient's budget"
            K, ph = k * k * cin, oh // 2
            x = torch.zeros(1, s, s, cin, dtype=torch.bfloat16, device=dev)
            wT = torch.zeros(cout, K + 8, dtype=torch.bfloat16, device=dev)
            pooled = torch.zeros(ph * ph * cout, dtype=torch.bfloat16, device=dev)
            am = torch.zeros(ph * ph * cout, dtype=torch.uint8, device=dev)
            dW, db = torch.zeros(K * cout, device=dev), torch.zeros(cout, device=dev)
            geo = dict(pad_top=pt, pad_left=pt, out_h=oh, out_w=oh)

            def wgrad():
                C.conv_first_wgrad(native.ptr(x), 1, s, s, cin, k, k, cout, native.ptr(pooled), native.ptr(pooled), native.ptr(am),
                                   R.ACT["relu"], native.ptr(dW), native.ptr(db), st, **geo)
            if ok:
                admitted += 1
                C.conv_first_fwd(native.ptr(x), 1, s, s, cin, k, k, cout, native.ptr(wT), wT.shape[1], 0, R.ACT["relu"],
                                 native.ptr(pooled), native.ptr(am), st, **geo)
                wgrad()
            elif over:
                refused_by_budget += 1
                with pytest.raises(RuntimeError, match=r"rc=-8"):
                    wgrad()
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    print(f"[conv-first] sweep: {admitted} admitted shapes launched, {refused_by_budget} refused past the wgrad budget")
    assert admitted > 100 and refused_by_budget > 20


# ------------------------------------------------------------------------------------------------------------------
# GPU: a first conv past the budget trains on the lowered path; every device gets its opt-in
# ------------------------------------------------------------------------------------------------------------------
# (relative Frobenius, max-abs / max|ref|) against the bf16-emulating step oracle, at about 3x what this test measured on
# an H100 80GB HBM3 (700 W power limit): 7.8e-6, 9.7e-6
LOWERED_TOL = (3e-5, 3e-5)


@pytest.mark.gpu
def test_first_conv_past_the_wgrad_budget_trains_lowered(monkeypatch):
    """64 x 64 x 3 input, 4 x 4 VALID conv to 16 channels, ReLU, 2 x 2 pool: its weight gradient would need 99,328 B of
    shared memory, so the step runs im2col + GEMM instead and matches the float64 step oracle."""
    import test_step_gradients as S

    name = "conv1_past_wgrad_budget"
    ir, lp = R.first_conv_plan(64, 64, 3, 4, 16, "valid")
    monkeypatch.setitem(S._MODEL_CACHE, name, (ir, lp, "y:0"))
    monkeypatch.setitem(S.MODELS, name, ({}, "onehot"))
    assert fused_first_conv(lp) is None
    w = S._weights(name)
    master, worker = S._worker(name, w)
    try:
        for B in (1, 7):
            X, Y = S._data(name, B, seed=B)
            got, loss, dbg, names = S._run_step(worker, B, X, Y, "staged")
            base = [nm.split("@")[0] for nm in names]
            assert "conv_first_fwd" not in base and "im2col" in base, names
            S._compare_step(f"{name} B={B}", lp, w, X, Y, got, loss, dbg, LOWERED_TOL)
    finally:
        master.close()


@pytest.mark.gpu
def test_every_device_opts_in(C):
    """The cnn geometry's weight gradient needs 52,800 B, past the 48 KiB default: the opt-in is a per-device setting,
    set when the module is first used on each device.  One process runs the forward and weight gradient on every
    visible device, each checked bit-exactly against float64."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    for d in range(torch.cuda.device_count()):
        with torch.cuda.device(d):
            _check(native.cuda_ext(), "cnn", 7, "relu", True, seed=d)
