"""float64 reference of the fused first convolution (csrc/conv.cu: conv_first_fwd_kernel, conv_first_wgrad_kernel) and
element-wise error bounds derived from their fp32 arithmetic, plus the launchers' shared-memory and dispatch formulas.
Device-agnostic: the CPU tests use it too.

Geometry (TensorFlow's): the conv output z [n, oh, ow, cout] is computed over the image padded with pad_top rows above,
pad_left columns to the left and the rest of the (oh + kh - 1) x (ow + kw - 1) frame below / right.  The 2x2 / stride-2
pool covers the oh // 2 x ow // 2 windows (an odd last row or column is never pooled); the recorded winner is the
position 0..3 (row-major in its window) of the FIRST maximum."""
import math

import torch

from sparkflow_b200.ops.layout import round_up

ACT = {None: 0, "relu": 1, "sigmoid": 2, "tanh": 3}
U = 2.0 ** -24                      # fp32 unit roundoff
U_BF16 = 2.0 ** -8                  # bf16 unit roundoff
THREADS = 256                       # kConv1Threads: n_grp * cout == THREADS for every cout the launchers take
MAX_SMEM = 96 * 1024                # kConv1MaxSmem


# ------------------------------------------------------------------------------------------------------------------
# the launchers' formulas (csrc/conv.cu: SF_CONV1_DISPATCH, conv_first_fwd_launch, conv_first_wgrad_launch)
# ------------------------------------------------------------------------------------------------------------------
def instance(kh, kw, cin):
    """the kernel template instance SF_CONV1_DISPATCH picks (0, 0, 0 = runtime shape)"""
    return (kh, kw, cin) if (kh, kw, cin) in ((5, 5, 1), (3, 3, 1), (3, 3, 3)) else (0, 0, 0)


def fwd_smem(kh, kw, cin, cout, oh, ow):
    """conv_first_fwd_launch: the runtime-shape instance's [K][cout] filter bank plus the padded image, fp32"""
    K = kh * kw * cin
    bank = K * cout if instance(kh, kw, cin) == (0, 0, 0) else 0
    return (bank + (oh + kh - 1) * (ow + kw - 1) * cin) * 4


def wgrad_smem(kh, kw, cin, cout, oh, ow):
    """conv_first_wgrad_launch: (bytes it asks for, staged?).  The padded image and the [n_grp][K + 1][cout] group
    reduction (the launch is refused above the cap), then the per-image dL/dz and argmax staging if it still fits."""
    K = kh * kw * cin
    base = ((oh + kh - 1) * (ow + kw - 1) * cin + THREADS * (K + 1)) * 4
    pc = (oh // 2) * (ow // 2) * cout
    staged = base + pc * 4 + (pc + 15) // 16 * 16
    return (staged, True) if staged <= MAX_SMEM else (base, False)


def fwd_parts(n, cout, oh, ow, sms):
    """conv_first_fwd_launch's split of an image over CTAs (`parts`) and its grid"""
    slots, n_grp, P = sms * 4, THREADS // cout, (oh // 2) * (ow // 2)
    parts, best = 1, 1e30
    for p in range(1, 9):
        items = n * p
        waves = (items + slots - 1) // slots
        util = items / slots if items < slots else 1.0
        cost = waves * ((P + n_grp * p - 1) // (n_grp * p) + 2.0) / util
        if cost < best:
            best, parts = cost, p
    return parts, min(n * parts, slots)


def wgrad_grid(n, sms):
    return max(1, min(n, 2 * sms))


def first_conv_plan(h, w, cin, k, cout, padding, act="relu"):
    """LayerPlan of a classifier whose first layer is a k x k conv of an h x w x cin image, then a 2x2 / 2 max-pool"""
    from sparkflow_b200.graph import tfcompat as tf
    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.graph_utils import build_graph
    from sparkflow_b200.models.compiler import compile_graph

    def fn():
        x = tf.placeholder(tf.float32, shape=[None, h * w * cin], name="x")
        y = tf.placeholder(tf.float32, shape=[None, 10], name="y")
        a = {"relu": tf.nn.relu, None: None}[act]
        c = tf.layers.conv2d(tf.reshape(x, shape=[-1, h, w, cin]), cout, k, padding=padding, activation=a)
        p = tf.layers.max_pooling2d(c, 2, 2)
        logits = tf.layers.dense(tf.layers.flatten(p), 10)
        tf.argmax(logits, 1, name="out")
        return tf.losses.softmax_cross_entropy(y, logits)

    ir = GraphIR.from_metagraph(build_graph(fn))
    return ir, compile_graph(ir, "x:0", "y:0")


def same_pads(k):
    """TF SAME at stride 1: (before, after)"""
    return (k - 1) // 2, k - 1 - (k - 1) // 2


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def operands(n, h, w, cin, kh, kw, cout, exact, seed, dev, lim=3):
    """x [n, h, w, cin] bf16, wT [cout, round_up(K, 8)] bf16 (row c = filter of channel c, k = (dy * kw + dx) * cin + ci;
    the pad columns hold 99, which no launch may read) and an fp32 bias [cout].  exact: integers in [-lim, lim] and an
    integer bias in [-8, 8], so every fp32 partial sum of the forward is exact; otherwise normal values scaled so that
    |z| stays around 1 and the activations are not saturated."""
    g = torch.Generator().manual_seed(seed)
    K = kh * kw * cin
    if exact:
        x = torch.randint(-lim, lim + 1, (n, h, w, cin), generator=g).float()
        wm = torch.randint(-lim, lim + 1, (K, cout), generator=g).float()
        bias = torch.randint(-8, 9, (cout,), generator=g).float()
    else:
        x = torch.randn(n, h, w, cin, generator=g)
        wm = torch.randn(K, cout, generator=g) / math.sqrt(K)
        bias = torch.randn(cout, generator=g) * 0.3
    wT = torch.full((cout, round_up(K, 8)), 99.0, dtype=torch.bfloat16)
    wT[:, :K] = wm.t().to(torch.bfloat16)
    return x.to(torch.bfloat16).to(dev), wT.to(dev), bias.to(dev)


def pool_grad(n, ph, pw, cout, exact, seed, dev, lim=3):
    """dL/d(pooled) [n, ph, pw, cout] bf16: integers in [-lim, lim] or normal values"""
    g = torch.Generator().manual_seed(seed + 1)
    v = torch.randint(-lim, lim + 1, (n, ph, pw, cout), generator=g).float() if exact else torch.randn(n, ph, pw, cout, generator=g)
    return v.to(torch.bfloat16).to(dev)


def filters(wT, kh, kw, cin):
    """the float64 filter bank W [K, cout] without the pad columns"""
    return wT[:, :kh * kw * cin].t().double()


# ------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------
def pad_image(x, kh, kw, pt, pl, oh, ow):
    """x [n, h, w, cin] -> float64 [n, oh + kh - 1, ow + kw - 1, cin] with the image at (pt, pl) in a zero frame"""
    n, h, w, cin = x.shape
    xp = torch.zeros(n, oh + kh - 1, ow + kw - 1, cin, dtype=torch.float64, device=x.device)
    xp[:, pt:pt + h, pl:pl + w] = x.double()
    return xp


def patches(xp, kh, kw, rows, cols, taps=None):
    """[n, rows, cols, K]: the input under each tap k = (ty * kw + tx) * cin + ci of the outputs (y, x) in rows x cols
    (ranges or strided slices of the conv output); `taps` replaces the tap order [(ty, tx), ...] (fault models)"""
    cin = xp.shape[3]
    taps = taps or [(ty, tx) for ty in range(kh) for tx in range(kw)]
    out = [xp[:, rows.start + ty:rows.stop + ty:rows.step, cols.start + tx:cols.stop + tx:cols.step] for ty, tx in taps]
    return torch.stack(out, 3).reshape(*out[0].shape[:3], len(taps) * cin)


def _act64(z, act):
    return {None: lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[act](z)


def forward(xp, W, bias, kh, kw, oh, ow, act):
    """float64 activation a = act(z) [n, oh, ow, cout] and the element-wise bound on the kernel's fp32 a:
      * z: the bias, then K fused multiply-adds, each rounding once: (K + 1) u of |bias| + sum_k |w_k x_k|;
      * sigmoid (1 / (1 + __expf(-z))): the slope <= 1/4 carries z's error, and __expf's (2 + 1.17 |z|) ulp, the add
        and the division stay below 2^-20 (1 + |z|) of the value;
      * tanhf: slope <= 1 carries z's error, plus 2^-20 (1 + |z|) absolutely (looser than tanhf's 2 ulp);
      * relu and none pass z's error on."""
    K = W.shape[0]
    P = patches(xp, kh, kw, slice(0, oh, 1), slice(0, ow, 1))
    b = bias.double() if bias is not None else torch.zeros(W.shape[1], dtype=torch.float64, device=W.device)
    z = P @ W + b
    e = (K + 1) * U * (P.abs() @ W.abs() + b.abs())
    if act == "sigmoid":
        a = torch.sigmoid(z)
        e = e / 4 + 2.0 ** -20 * (1 + z.abs()) * a
    elif act == "tanh":
        a = torch.tanh(z)
        e = e + 2.0 ** -20 * (1 + z.abs())
    else:
        a = _act64(z, act)
    return a, e


def windows(t, ph, pw):
    """[n, oh, ow, c] -> [n, ph, pw, c, 4]: the 2x2 windows, positions in row-major order"""
    n, _, _, c = t.shape
    return t[:, :2 * ph, :2 * pw].reshape(n, ph, 2, pw, 2, c).permute(0, 1, 3, 5, 2, 4).reshape(n, ph, pw, c, 4)


def first_max(v):
    """index of the first maximum along the last dimension (the kernel's strict `>` scan)"""
    m = v.max(-1, keepdim=True).values
    idx = torch.full(v.shape[:-1], 3, dtype=torch.long, device=v.device)
    for k in (2, 1, 0):
        idx = torch.where(v[..., k] == m[..., 0], torch.full_like(idx, k), idx)
    return idx


def pool(a, ph, pw):
    """float64 pooled maximum and its first-maximum winner"""
    v = windows(a, ph, pw)
    idx = first_max(v)
    return v.gather(-1, idx.unsqueeze(-1)).squeeze(-1), idx


def check_forward(tag, a, e, pooled, argmax, exact):
    """The kernel's pooled [n, ph, pw, cout] bf16 and argmax uint8 against the float64 activation a and its bound e.
    exact (integer operands, none / relu): both bit-equal to bf16(first maximum) and its position.  Otherwise the
    recorded winner's activation is within the two roundings' bounds of its window maximum, and pooled is that
    activation up to its bound and one bf16 rounding.  With integer operands an activation tied in float64 is tied in
    the kernel too, so the recorded winner is never preceded by one equal to it.  Returns the number of windows whose
    maximum is tied."""
    n, ph, pw, cout = pooled.shape
    v, ve = windows(a, ph, pw), windows(e, ph, pw)
    best, first = pool(a, ph, pw)
    am = argmax.long()
    assert int(am.max()) <= 3, f"{tag}: argmax outside its window"
    ties = int(((v == best.unsqueeze(-1)).sum(-1) > 1).sum())
    if exact:
        bad = int((am != first).sum())
        assert bad == 0, f"{tag}: {bad} winners are not the first maximum of their window"
        want = best.float().to(torch.bfloat16)
        bad = int((pooled != want).sum())
        assert bad == 0, f"{tag}: {bad} pooled values differ from bf16(float64 maximum)"
        return ties
    win = v.gather(-1, am.unsqueeze(-1)).squeeze(-1)
    slack = ve.max(-1).values * 2
    bad = int((win < best - slack).sum())
    assert bad == 0, f"{tag}: {bad} recorded winners are below their window maximum by more than the bound"
    we = ve.gather(-1, am.unsqueeze(-1)).squeeze(-1)
    d = (pooled.double() - win).abs()
    lim = we + U_BF16 * (win.abs() + we)
    assert bool((d <= lim).all()), f"{tag}: pooled value off by {float((d / lim.clamp_min(1e-300)).max()):.2f} x its bound"
    return ties


def check_tie_rule(tag, a, argmax):
    """integer operands: no window position before the recorded winner holds the same float64 activation"""
    n, ph, pw, cout = argmax.shape
    v = windows(a, ph, pw)
    am = argmax.long()
    win = v.gather(-1, am.unsqueeze(-1))
    pos = torch.arange(4, device=a.device)
    earlier_tie = ((v == win) & (pos < am.unsqueeze(-1))).any(-1)
    assert not bool(earlier_tie.any()), f"{tag}: {int(earlier_tie.sum())} windows record a later one of tied maxima"


# ------------------------------------------------------------------------------------------------------------------
# weight gradient
# ------------------------------------------------------------------------------------------------------------------
def dact64(pooled, act):
    """act' at the STORED bf16 pooled value, as the kernel takes it (pool_dact in csrc/conv.cu)"""
    a = pooled.double()
    if act == "relu":
        return (a > 0).double()
    if act == "sigmoid":
        return a * (1 - a)
    if act == "tanh":
        return 1 - a * a
    return torch.ones_like(a)


def wgrad(xp, gz, argmax, kh, kw, taps=None, origin=False):
    """float64 dW [K, cout], db [cout] and sum_{img, p} |gz x| [K, cout] (for the bound) of dL/dz = gz [n, ph, pw, cout]
    at the recorded winners.  `taps` / `origin` (every winner at its window's origin) model faults."""
    n, ph, pw, cout = gz.shape
    K = xp.shape[3] * (len(taps) if taps else kh * kw)
    dW = torch.zeros(K, cout, dtype=torch.float64, device=xp.device)
    T = torch.zeros_like(dW)
    am = torch.zeros_like(argmax, dtype=torch.long) if origin else argmax.long()
    for q in range(4):
        dy, dx = q >> 1, q & 1
        sel = (gz * (am == q)).reshape(-1, cout)
        if not bool(sel.ne(0).any()):
            continue
        P = patches(xp, kh, kw, slice(dy, dy + 2 * ph, 2), slice(dx, dx + 2 * pw, 2), taps).reshape(-1, K)
        dW += P.t() @ sel
        T += P.abs().t() @ sel.abs()
    return dW, gz.sum((0, 1, 2)), T


def wgrad_bound(gz, T, dW0, db0, n, cout, oh, ow, sms):
    """Element-wise bounds of the kernel's dW and db (accumulated onto dW0, db0):
      * gz = g * act'(pooled) in fp32: act' (at most two roundings) and the product: 3u relative;
      * each thread (channel c, group grp) chains its fmas over every pixel p = grp (mod n_grp) of every image its CTA
        takes: L = ceil(n / grid) * ceil(P / n_grp) roundings;
      * the n_grp group partials are added in shared memory (n_grp roundings), then one atomic per CTA onto the start
        value (grid roundings).
    Every rounding is of a partial sum no larger than |start| + sum |terms|."""
    n_grp, P = THREADS // cout, (oh // 2) * (ow // 2)
    grid = wgrad_grid(n, sms)
    L = -(-n // grid) * -(-P // n_grp)
    m = L + n_grp + grid + 3
    gabs = gz.abs().sum((0, 1, 2))
    eW = 1.01 * m * U * (T + dW0.double().abs())
    eb = 1.01 * m * U * (gabs + db0.double().abs())
    return eW, eb


def fraction(got, ref, bound):
    """worst |got - ref| / bound (0 where both are 0)"""
    d = (got.double() - ref).abs()
    return float((d / bound.clamp_min(1e-300)).max())
