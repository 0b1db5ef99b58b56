"""LayerPlan -> native step plan (list of sm_90a kernel launches, later a CUDA graph).

Supported layer grammar (anything else is reported as UnsupportedGraph and handled by the generic engine):

    input -> [reshape] -> (conv [maxpool])* -> [flatten] -> dense+ -> loss

conv: NHWC, VALID or SAME padding, stride (sh, sw); maxpool: window up to 4x4, stride (sh, sw), VALID or SAME (TF geometry,
see models/compiler.py).  A conv without a pool after it feeds the next conv or the flatten directly.

Data-flow conventions (all activations bf16, all accumulation fp32):

* dense layer i consumes ``a_i`` [B, ld] (A operand) and the published ``W_i^T`` [out, ld] (B operand);
  its epilogue adds bias, applies the activation and writes ``a_{i+1}`` plus ``a_{i+1}^T`` (the K-major
  operand of the next layer's wgrad).  The last dense layer's epilogue also computes the loss and dL/dz.
* conv is im2col (patches + patches^T; out-of-image taps of a padded conv read zero) followed by the same GEMM; NHWC
  activations are exactly the row-major GEMM output, so no layout conversion exists anywhere.
* max-pool: 2x2 / stride 2 without padding runs on the dedicated kernels (SAME on even sizes included), every other
  geometry on the general window kernels.
* backward: ``dgrad`` GEMMs run on the main branch of the graph, ``wgrad`` GEMMs (which only feed the push)
  alternate between two side branches, except the first layer's, which the push waits for: it runs on the main
  branch; bias gradients come out of epilogues / the pool-backward kernel (or, for a conv with no pool after it, the
  activation-gradient kernel); every gradient lands in the flat fp32 buffer the push kernel consumes.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import os
import struct

import torch

from ..models.compiler import ACT_IDS, Layer, LayerPlan, UnsupportedGraph
from ..ops import native
from ..ops.layout import round_up


@dataclass
class BuiltPlan:
    plan: Any
    x_stage: torch.Tensor
    y_stage: Optional[torch.Tensor]
    loss_out: torch.Tensor
    result: Optional[torch.Tensor] = None
    keep: List[Any] = field(default_factory=list)
    debug: Optional[Dict[int, Dict[str, Any]]] = None     # per layer index: intermediate buffers (tests / tools)


def pool_fast_path(l: Layer) -> bool:
    """A 2x2 / stride-2 max-pool with zero effective padding runs on the dedicated 2x2 kernels."""
    return l.ksize == (2, 2) and l.strides == (2, 2) and not any(l.pads)


def _kmajor_geometry_ok(layers: List[Layer]) -> bool:
    """The K-major weight-gradient path (SPARKFLOW_WGRAD_MN=0) needs transposed copies that only the VALID stride-1 conv
    followed by the 2x2 / stride-2 pool kernels write."""
    for i, l in enumerate(layers):
        if l.kind == "conv":
            if l.strides != (1, 1) or any(l.pads) or i + 1 >= len(layers) or layers[i + 1].kind != "pool":
                return False
        elif l.kind == "pool" and not pool_fast_path(l):
            return False
    return True


def check_grammar(lp: LayerPlan) -> None:
    """Raise UnsupportedGraph unless the layer sequence matches the grammar above."""
    kinds = [l.kind for l in lp.layers]
    i = 0
    if i < len(kinds) and kinds[i] == "reshape":
        i += 1
    saw_conv = False
    while i < len(kinds) and kinds[i] == "conv":
        saw_conv = True
        i += 1
        if i < len(kinds) and kinds[i] == "pool":
            i += 1
    if i < len(kinds) and kinds[i] == "reshape":
        i += 1
    n_dense = 0
    while i < len(kinds) and kinds[i] == "dense":
        n_dense += 1
        i += 1
    if i != len(kinds) or n_dense == 0:
        raise UnsupportedGraph(f"layer sequence {kinds} is outside the compiled plan grammar "
                               "(input -> [reshape] -> (conv [maxpool])* -> [flatten] -> dense+)")
    for l in lp.layers:
        if l.kind == "conv":
            if l.out_shape[2] % 8:
                raise UnsupportedGraph("conv output channels must be a multiple of 8")
            if l.act not in ACT_IDS:
                raise UnsupportedGraph(f"conv activation {l.act}")
    if saw_conv and lp.input_dim % 8:
        raise UnsupportedGraph("image inputs need a feature count that is a multiple of 8")
    if saw_conv and not use_mn_possible(True) and not _kmajor_geometry_ok(lp.layers):
        raise UnsupportedGraph("SPARKFLOW_WGRAD_MN=0 (K-major weight gradients) covers only VALID stride-1 convs each followed by a "
                               "2x2 / stride-2 max-pool")


def fused_first_conv(lp: LayerPlan) -> Optional[int]:
    """Index of the network's first trainable layer when it is a small stride-1 convolution directly followed by a 2x2 /
    stride-2 max-pool without padding (K = kh * kw * cin <= 64, 8..64 output channels, the zero-padded image within 64 KiB
    of fp32): that pair runs as ONE direct CUDA-core kernel forward and ONE backward (csrc/conv.cu: conv_first_fwd /
    conv_first_wgrad) instead of im2col + a K-padded GEMM + a pooling pass."""
    if os.environ.get("SPARKFLOW_FUSED_CONV1", "1") == "0":
        return None
    layers = lp.layers
    trainable = [i for i, l in enumerate(layers) if l.kind in ("dense", "conv")]
    if not trainable:
        return None
    i = trainable[0]
    l = layers[i]
    if l.kind != "conv" or i + 1 >= len(layers) or layers[i + 1].kind != "pool" or not pool_fast_path(layers[i + 1]):
        return None
    if l.strides != (1, 1):
        return None
    cin, cout = l.in_shape[2], l.out_shape[2]
    if l.ksize[0] * l.ksize[1] * cin > 64 or cout not in (8, 16, 32, 64) or l.act not in (None, "Relu", "Sigmoid", "Tanh"):
        return None
    if (l.out_shape[0] + l.ksize[0] - 1) * (l.out_shape[1] + l.ksize[1] - 1) * cin * 4 > 64 * 1024:
        return None
    return i


def act_arg(l: Layer) -> int:
    """The ``act`` argument of the stand-alone backward / loss kernels for layer ``l``: its SfAct in the low 32 bits and
    the fp32 bits of a leaky ReLU's alpha in the high 32 (csrc/runtime.cpp, launch::act_kind / act_alpha)."""
    return ACT_IDS[l.act] | (struct.unpack("<I", struct.pack("<f", l.act_alpha))[0] << 32)


_LOSS_MODES = {"softmax_xent": 1, "mse": 2, "sigmoid_xent": 3, "sparse_softmax_xent": 4}     # SfLossMode (csrc/sf_api.h)


def loss_mode(kind: Optional[str]) -> int:
    """the fused-loss GEMM epilogue's head for LayerPlan loss kind ``kind``"""
    if kind not in _LOSS_MODES:
        raise UnsupportedGraph(f"no fused loss head for loss kind {kind!r}")
    return _LOSS_MODES[kind]


def _split_k(tiles: int, kblocks: int) -> int:
    if kblocks < 16:
        return 1
    return max(1, min(native.num_sms() // max(tiles, 1), kblocks // 4))


def use_mn_possible(train: bool) -> bool:
    """MN-major weight gradients (no transposed activation copies) are used unless switched off; forward-only plans never
    need transposes."""
    return not train or os.environ.get("SPARKFLOW_WGRAD_MN", "1") == "1"


def build_prep(worker, B: int, inputs: Dict[str, Any], resident: Optional[Dict[str, Any]] = None):
    """Plan that prepares input set ``inputs`` (see ``build``) for one training step, run before the step's graph on the
    stream that stages the minibatch.  DMA staging: cast (+ transpose) of the fp32 rows already copied into ``x32``.
    ``resident``: dict(x, y) device tensors holding the whole partition in HBM: gather + cast of the rows whose ids are in
    the returned ``idx`` buffer, and a row gather of the labels (or, for autoencoders, of the fp32 target rows).
    Returns (plan, idx or None)."""
    C, lp = worker.C, worker.plan
    P = native.ptr
    D = lp.input_dim
    a0, a0T, x32, y = inputs["a0"], inputs["a0T"], inputs["x32"], inputs["y"]
    ldT = a0T.shape[1] if a0T is not None else 0
    plan = C.Plan()
    if resident is None:
        plan.add_cast_transpose(P(x32), D, 0, P(a0), a0.shape[1], P(a0T), ldT, B, D)
        return plan, None
    idx = torch.zeros(B, dtype=torch.int32, device=worker.device)
    xr, yr = resident["x"], resident["y"]
    plan.add_cast_transpose(P(xr), xr.shape[1], P(idx), P(a0), a0.shape[1], P(a0T), ldT, B, D)
    if lp.target_is_input:
        plan.add_gather_rows(P(xr), xr.shape[1], P(idx), P(x32), D, B, D)
    if y is not None:
        plan.add_gather_rows(P(yr), yr.shape[1], P(idx), P(y), y.shape[1], B, y.shape[1])
    return plan, idx


def build(worker, B: int, *, train: bool, with_pull: bool, with_push: bool = True, upto: Optional[int] = None,
          post: Optional[str] = None, with_loss: bool = False, inputs: Optional[Dict[str, Any]] = None) -> BuiltPlan:
    """``train``: full step (fwd + loss + bwd + push).  Otherwise forward up to dense index ``upto``
    (None = last) producing an fp32 result (+ArgMax), or forward + loss only when ``with_loss``.

    ``inputs``: dict(x32, a0, a0T, y) already holding this step's minibatch (fp32 rows, bf16 operands, labels) when the
    graph starts - filled by ``build_prep``'s plan - so the graph has no cast kernel and starts with the pull."""
    C, dev, lay, lp = worker.C, worker.device, worker.layout, worker.plan
    check_grammar(lp)
    P = native.ptr
    bf16, f32 = torch.bfloat16, torch.float32
    keep: List[Any] = []

    def zeros(*shape, dtype=bf16):
        t = torch.zeros(*shape, dtype=dtype, device=dev)
        keep.append(t)
        return t

    ldB = round_up(B, 8)
    D = lp.input_dim
    need_labels = (train or with_loss) and not lp.target_is_input
    if inputs is not None:
        x_stage, y_stage = inputs["x32"], inputs["y"]
    else:
        x_stage = zeros(B, D, dtype=f32)
        y_stage = zeros(B, lp.label_dim, dtype=f32) if need_labels else None
    done_dev = None
    if train and os.environ.get("SPARKFLOW_DEVICE_LOSS") != "1":
        # training steps hand their loss to the host with a zero-copy store from the last kernel (pinned, device-mapped):
        # word 0 = loss, word 1 = completion sequence number (only written when a done counter is attached)
        loss_out = torch.zeros(2, dtype=f32).pin_memory()
        keep.append(loss_out)
        done_dev = zeros(1, dtype=torch.int32)
    else:
        loss_out = zeros(1, dtype=f32)
    wsrc = worker._weight_src()
    plan = C.Plan()
    branches = worker.use_branches and train
    sharded = bool(getattr(worker, "sharded", False))
    do_pull = with_pull and (worker.pull_mode != "direct" or lay.vec_count > 0)
    fuse_ryw = False
    if sharded:
        # the step always starts with the read-your-writes wait (it also protects the mailboxes the wgrad epilogues
        # are about to overwrite); the seqlock snapshot is only taken when this step really pulls (lock mode).
        # Hogwild training steps fuse the wait into their first GEMM instead (no pull kernel at all).
        do_pull = bool(train or with_pull)
        fuse_ryw = bool(train and getattr(worker, "fuse_ryw", False))
        if fuse_ryw:
            do_pull = False
    fused_conv = fused_first_conv(lp) if use_mn_possible(train) else None
    if fused_conv is not None:
        fuse_ryw = False             # the first weight reader is the direct conv kernel: keep the stand-alone wait
        if sharded:
            do_pull = bool(train or with_pull)
    ryw_pending = [fuse_ryw]

    def ryw_args() -> Dict[str, Any]:
        """dict entries for the first weight-reading GEMM of the step (consumed once)"""
        if ryw_pending[0]:
            ryw_pending[0] = False
            return dict(ryw=P(worker.ryw_dev))
        return {}

    def add_pull_op():
        if sharded:
            plan.add_sync_pull(worker._sync_pull_args(copy=with_pull))
        else:
            plan.add_pull(worker._pull_args(), P(worker.sync_pull), 0)

    layers = lp.layers
    dense_ids = [i for i, l in enumerate(layers) if l.kind == "dense"]
    last_dense_pos = len(dense_ids) - 1 if upto is None else upto
    stop_layer = dense_ids[last_dense_pos]
    trainable = [i for i, l in enumerate(layers) if l.kind in ("dense", "conv")]
    first_trainable = trainable[0]

    # ---------------- pull || input cast ----------------
    # with `inputs` the operands are ready when the graph starts: the pull heads the main branch and the first GEMM
    # follows it over a programmatic edge (a join would be a full-completion edge).  The sharded snapshot pull keeps the
    # join: it waits for the shard appliers and lets its successors pre-launch before that wait.
    overlap_pull = do_pull and branches and (inputs is None or sharded)
    if overlap_pull:
        plan.fork(1)
        plan.branch(1)
        add_pull_op()
        plan.branch(0)
    elif do_pull:
        add_pull_op()
    first_is_dense = layers[first_trainable].kind == "dense"
    # weight gradients read the row-major activation / dz buffers directly (MN-major wgmma operands): no transposed copy
    # of any activation, gradient or im2col matrix is ever written.
    use_mn = bool(train and use_mn_possible(train))
    if inputs is not None:
        a0, a0T = inputs["a0"], inputs["a0T"]
    else:
        a0 = zeros(B, round_up(D, 8))
        a0T = zeros(D, ldB) if (train and first_is_dense and not use_mn) else None
        plan.add_cast_transpose(P(x_stage), D, 0, P(a0), a0.shape[1], P(a0T), ldB if a0T is not None else 0, B, D)
    if overlap_pull:
        plan.join(1)

    # ---------------- forward ----------------
    # `cur` describes the activation entering the next layer
    cur: Dict[str, Any] = dict(kind="flat", buf=a0, bufT=a0T, feat=D, ld=a0.shape[1])
    rec: Dict[int, Dict[str, Any]] = {}        # per-layer tensors needed by backward
    gemms: List[Any] = []

    def emit(g, name: str, on_side: bool = False) -> None:
        """Add a GEMM to the plan as its own launch, optionally on a wgrad branch."""
        gemms.append(g)
        if on_side:
            side(lambda: plan.add_gemm(g, name))
        else:
            plan.add_gemm(g, name)

    def wgrad_on_side(i: int) -> bool:
        """The first trainable layer's wgrad is the last GEMM of the step and the only one the push still waits for: it
        runs on the main branch right after the dgrad that produces its operand, and the push follows it over a
        programmatic edge.  Sharded steps keep it on a side branch, beside the post of the bias-gradient tail."""
        return i != first_trainable or sharded

    out_f32 = None
    dz_last = dzT_last = None
    fuse_loss = False
    target = x_stage if lp.target_is_input else y_stage
    for i, l in enumerate(layers):
        if i > stop_layer:
            break
        if l.kind == "reshape":
            if len(l.out_shape) == 3:                              # flat -> image (NHWC view of the same memory)
                if cur["ld"] != cur["feat"]:
                    raise UnsupportedGraph("reshape to an image needs an unpadded feature row")
                cur = dict(kind="img", buf=cur["buf"], shape=l.out_shape)
            else:                                                   # flatten: image -> flat view
                h, w, c = cur["shape"]
                cur = dict(kind="flat", buf=cur["buf"], bufT=cur.get("flatT"), feat=h * w * c, ld=h * w * c)
            continue
        if l.kind == "conv" and i == fused_conv:
            # first conv + bias + activation + 2x2 max-pool as ONE direct kernel: only the pooled tensor is written
            h, w, cin = cur["shape"]
            kh, kw = l.ksize
            oh, ow, cout = l.out_shape
            ph, pw = oh // 2, ow // 2
            ks, bs = lay.by_name(l.kernel), (lay.by_name(l.bias) if l.bias else None)
            pooled = zeros(B, ph * pw * cout)
            argmax = zeros(B, ph * pw * cout, dtype=torch.uint8)
            plan.add_conv_first_fwd(P(cur["buf"]), B, h, w, cin, kh, kw, cout, P(wsrc) + ks.wt_off * 2, ks.wt_ld,
                                    worker._bias_ptr(bs) if bs else 0, ACT_IDS[l.act], P(pooled), P(argmax), l.pads[0], l.pads[2], oh, ow)
            rec[i] = dict(fused=True, x=cur["buf"], in_shape=(h, w, cin), pooled=pooled, argmax=argmax)
            cur = dict(kind="img", buf=pooled, shape=(ph, pw, cout), flatT=None, fused_pool=i)
            continue
        if l.kind == "pool" and cur.get("fused_pool") is not None:
            rec[i] = dict(fused=True, conv=cur.pop("fused_pool"))
            continue
        if l.kind == "conv":
            h, w, cin = cur["shape"]
            kh, kw = l.ksize
            oh, ow, cout = l.out_shape
            M, K = B * oh * ow, kh * kw * cin
            ldK, ldM = round_up(K, 8), round_up(M, 8)
            patches = zeros(M, ldK)
            patchesT = zeros(K, ldM) if (train and not use_mn) else None
            plan.add_im2col(P(cur["buf"]), B, h, w, cin, kh, kw, P(patches), ldK, P(patchesT), ldM if patchesT is not None else 0,
                            l.strides[0], l.strides[1], l.pads[0], l.pads[2], oh, ow)
            ks, bs = lay.by_name(l.kernel), (lay.by_name(l.bias) if l.bias else None)
            act_out = zeros(M, cout)
            g = C.Gemm(dict(a=P(patches), lda=ldK, b=P(wsrc) + ks.wt_off * 2, ldb=ks.wt_ld, M=M, N=cout, K=K,
                            bias=worker._bias_ptr(bs) if bs else 0, act=ACT_IDS[l.act], act_alpha=l.act_alpha, out_bf16=P(act_out), ld_bf16=cout,
                            a_evict_first=1, **ryw_args()))
            gemms.append(g)
            plan.add_gemm(g, f"conv{i}")
            rec[i] = dict(patches=patches, patchesT=patchesT, act_out=act_out, in_shape=(h, w, cin), M=M, K=K, ldM=ldM, ldK=ldK)
            cur = dict(kind="img", buf=act_out, shape=(oh, ow, cout), conv=i)
            continue
        if l.kind == "pool":
            h, w, c = cur["shape"]
            oh, ow = l.out_shape[0], l.out_shape[1]
            pooled = zeros(B, oh * ow * c)
            argmax = zeros(B, oh * ow * c, dtype=torch.uint8)
            flatT = None
            if pool_fast_path(l):
                nxt_dense = (i + 2 < len(layers) and layers[i + 1].kind == "reshape" and layers[i + 2].kind == "dense")
                flatT = zeros(oh * ow * c, ldB) if (train and nxt_dense and not use_mn) else None
                plan.add_maxpool_fwd(P(cur["buf"]), B, h, w, c, P(pooled), P(argmax), P(flatT), ldB if flatT is not None else 0)
            else:
                plan.add_maxpool_gen_fwd(P(cur["buf"]), B, h, w, c, l.ksize[0], l.ksize[1], l.strides[0], l.strides[1], l.pads[0], l.pads[2],
                                         oh, ow, P(pooled), P(argmax))
            rec[i] = dict(argmax=argmax, in_shape=(h, w, c), conv=cur.get("conv"), pooled=pooled)
            cur = dict(kind="img", buf=pooled, shape=(oh, ow, c), flatT=flatT)
            continue
        # ---- dense ----
        ks, bs = lay.by_name(l.kernel), (lay.by_name(l.bias) if l.bias else None)
        last = i == stop_layer
        d = dict(a=P(cur["buf"]), lda=cur["ld"], b=P(wsrc) + ks.wt_off * 2, ldb=ks.wt_ld, M=B, N=ks.cols, K=ks.rows,
                 bias=worker._bias_ptr(bs) if bs else 0, act=ACT_IDS[l.act], act_alpha=l.act_alpha, **ryw_args())
        drop = None
        if l.dropout_keep:
            # fused Philox dropout: the mask is a function of (row, column, step counter of this plan, layer) under a
            # seed that also mixes in the worker index and the address of the plan's step counter
            seed = (int(os.environ.get("SPARKFLOW_DROPOUT_SEED", "20260921")) ^ (0x9E3779B9 * (worker.worker_index + 1))
                    ^ ((P(done_dev) >> 4) if done_dev is not None else 0)) & 0xFFFFFFFF
            d.update(drop_keep=float(l.dropout_keep), drop_seed=seed, drop_stream=i, drop_ctr=P(done_dev) if done_dev is not None else 0)
            drop = dict(keep=float(l.dropout_keep), seed=seed, stream=i, ctr=done_dev)
        rec[i] = dict(a_in=cur["buf"], a_in_ld=cur["ld"], a_inT=cur.get("bufT"), drop=drop)
        if last:
            # the element-wise heads take any width; a softmax row (dense or sparse labels) must fit one 32-column
            # epilogue chunk
            fuse_loss = train and worker.fuse_loss and (lp.loss not in ("softmax_xent", "sparse_softmax_xent") or ks.cols <= 32)
            if fuse_loss:
                dz_last, dzT_last = zeros(B, round_up(ks.cols, 8)), (None if use_mn else zeros(ks.cols, ldB))
                db = P(worker.grads) + bs.offset * 4 if bs else 0
                d.update(loss_mode=loss_mode(lp.loss), target=P(target), ld_target=target.shape[1],
                         loss=P(worker.loss_acc), out_bf16=P(dz_last), ld_bf16=dz_last.shape[1], outT_bf16=P(dzT_last),
                         ld_t=ldB if dzT_last is not None else 0, colsum=db)
            else:
                out_f32 = zeros(B, ks.cols, dtype=f32)
                d.update(out_f32=P(out_f32), ld_f32=ks.cols)
            g = C.Gemm(d)
            emit(g, f"fwd{i}" + ("+loss" if fuse_loss else ""))
            rec[i].update(N=ks.cols, fwd=g)
            break
        nxt = zeros(B, round_up(ks.cols, 8))
        nxtT = zeros(ks.cols, ldB) if (train and not use_mn) else None
        d.update(out_bf16=P(nxt), ld_bf16=nxt.shape[1], outT_bf16=P(nxtT), ld_t=ldB if nxtT is not None else 0)
        g = C.Gemm(d)
        emit(g, f"fwd{i}")
        rec[i]["fwd"] = g
        cur = dict(kind="flat", buf=nxt, bufT=nxtT, feat=ks.cols, ld=nxt.shape[1])

    result = None
    last_l = layers[stop_layer]
    n_out = lay.by_name(last_l.kernel).cols

    def add_loss(loss, dz, ld_dz, dzT, ld_t, db):
        """stand-alone loss kernel on the fp32 output of the last layer (pointers 0: not written)"""
        args = (P(out_f32), n_out, P(target), target.shape[1])
        if lp.loss == "softmax_xent":
            plan.add_softmax_xent(*args, loss, dz, ld_dz, dzT, ld_t, db, B, n_out)
        elif lp.loss == "sparse_softmax_xent":
            # a label row of width 1 < n_out: the binding reads it as one class index per row
            plan.add_softmax_xent(P(out_f32), n_out, P(target), 1, loss, dz, ld_dz, dzT, ld_t, db, B, n_out)
        elif lp.loss == "sigmoid_xent":
            plan.add_sigmoid_xent(*args, loss, dz, ld_dz, dzT, ld_t, db, B, n_out)
        elif lp.loss == "mse":
            plan.add_mse(*args, act_arg(last_l), loss, dz, ld_dz, dzT, ld_t, db, B, n_out)
        else:
            raise UnsupportedGraph(f"no loss kernel for loss kind {lp.loss!r}")

    if not train:
        if with_loss:
            add_loss(P(loss_out), 0, 0, 0, 0, 0)
        elif post == "ArgMax":
            result = zeros(B, dtype=f32)
            plan.add_argmax(P(out_f32), n_out, P(result), B, n_out)
        else:
            result = out_f32
        keep.append(gemms)
        return BuiltPlan(plan, x_stage, y_stage, loss_out, result, keep)

    # ---------------- loss (when not fused) ----------------
    bs_last = lay.by_name(last_l.bias) if last_l.bias else None
    if not fuse_loss:
        dz_last, dzT_last = zeros(B, round_up(n_out, 8)), (None if use_mn else zeros(n_out, ldB))
        db = P(worker.grads) + bs_last.offset * 4 if bs_last else 0
        add_loss(P(worker.loss_acc), P(dz_last), dz_last.shape[1], P(dzT_last), ldB if dzT_last is not None else 0, db)

    # ---------------- backward ----------------
    n_side = [0]

    def side(fn):
        """run `fn` (which adds ops) on a wgrad branch: branches 2 and 1 alternate, so no wgrad queues behind the previous
        one"""
        if branches:
            b = 2 - n_side[0] % 2
            n_side[0] += 1
            plan.fork(b)
            plan.branch(b)
        fn()
        plan.branch(0)

    # gradient flowing into the current layer from above
    g_dz, g_dzT = dz_last, dzT_last              # wrt the pre-activation of the layer being processed (dense)
    g_img = None                                  # wrt the pooled output (feeds maxpool_bwd)
    for i in range(stop_layer, -1, -1):
        l = layers[i]
        if l.kind == "dense":
            ks = lay.by_name(l.kernel)
            r = rec[i]
            if use_mn:
                # dW = a_in^T . dz straight from the row-major buffers (both operands MN-major)
                wd = dict(a=P(r["a_in"]), lda=r["a_in_ld"], b=P(g_dz), ldb=g_dz.shape[1], M=ks.rows, N=ks.cols, K=B, mn_major=1)
            else:
                if r["a_inT"] is None:
                    raise UnsupportedGraph("dense layer input has no transposed copy")
                wd = dict(a=P(r["a_inT"]), lda=ldB, b=P(g_dzT), ldb=ldB, M=ks.rows, N=ks.cols, K=B)
            if sharded:
                wd.update(worker.route_args(ks))          # push fused into the epilogue: tiles go to the owners' mailboxes
            else:
                wd.update(out_f32=P(worker.grads) + ks.offset * 4, ld_f32=ks.cols)
            wg = C.Gemm(wd)
            r["wgrad"] = wg
            emit(wg, f"wgrad{i}", on_side=wgrad_on_side(i))
            if i == first_trainable:
                break
            prev = layers[i - 1]
            if prev.kind == "dense":
                pb = lay.by_name(prev.bias) if prev.bias else None
                ndz, ndzT = zeros(B, r["a_in_ld"]), (None if use_mn else zeros(ks.rows, ldB))
                dd = dict(a=P(g_dz), lda=g_dz.shape[1], b=P(wsrc) + ks.w_off * 2, ldb=ks.w_ld, M=B, N=ks.rows, K=ks.cols,
                          aux=P(r["a_in"]), ld_aux=r["a_in_ld"], aux_act=ACT_IDS[prev.act], aux_act_alpha=prev.act_alpha, aux_keep=float(prev.dropout_keep or 0.0), out_bf16=P(ndz),
                          ld_bf16=ndz.shape[1], outT_bf16=P(ndzT), ld_t=ldB if ndzT is not None else 0,
                          colsum=P(worker.grads) + pb.offset * 4 if pb else 0)
                dg = C.Gemm(dd)
                emit(dg, f"dgrad{i}")
                r["dgrad"] = dg
                g_dz, g_dzT = ndz, ndzT
            else:                                  # flatten over an image: gradient wrt the pooled tensor / the conv activation
                g_img = zeros(B, ks.rows)
                dg = C.Gemm(dict(a=P(g_dz), lda=g_dz.shape[1], b=P(wsrc) + ks.w_off * 2, ldb=ks.w_ld, M=B, N=ks.rows, K=ks.cols,
                                 out_bf16=P(g_img), ld_bf16=ks.rows))
                gemms.append(dg)
                plan.add_gemm(dg, f"dgrad{i}")
            continue
        if l.kind == "reshape":
            continue
        if l.kind == "pool" and rec[i].get("fused"):
            ci = rec[i]["conv"]
            conv_l, cr = layers[ci], rec[ci]
            ks = lay.by_name(conv_l.kernel)
            cb = lay.by_name(conv_l.bias) if conv_l.bias else None
            h, w, cin = cr["in_shape"]
            plan.add_conv_first_wgrad(P(cr["x"]), B, h, w, cin, conv_l.ksize[0], conv_l.ksize[1], ks.cols, P(g_img), P(cr["pooled"]),
                                      P(cr["argmax"]), ACT_IDS[conv_l.act], P(worker.grads) + ks.offset * 4,
                                      P(worker.grads) + cb.offset * 4 if cb else 0, conv_l.pads[0], conv_l.pads[2], conv_l.out_shape[0],
                                      conv_l.out_shape[1])
            break                                  # it is the first trainable layer: nothing below needs a gradient
        if l.kind == "pool":
            r = rec[i]
            ci = r["conv"]
            conv_l, cr = layers[ci], rec[ci]
            h, w, c = r["in_shape"]
            cb = lay.by_name(conv_l.bias) if conv_l.bias else None
            need_dz = ci != first_trainable or use_mn   # conv dgrad (and the MN-major wgrad) read the row-major dz
            dzc = zeros(cr["M"], c) if need_dz else None
            dzcT = None if use_mn else zeros(c, cr["ldM"])
            if pool_fast_path(l):
                plan.add_maxpool_bwd(P(g_img), P(r["argmax"]), B, h, w, c, P(cr["act_out"]), act_arg(conv_l), P(dzc), c if need_dz else 0,
                                     P(dzcT), cr["ldM"] if dzcT is not None else 0, P(worker.grads) + cb.offset * 4 if cb else 0)
            else:                                   # check_grammar keeps general pools off the K-major path: dz is row-major only
                plan.add_maxpool_gen_bwd(P(g_img), P(r["argmax"]), B, h, w, c, l.ksize[0], l.ksize[1], l.strides[0], l.strides[1], l.pads[0],
                                         l.pads[2], l.out_shape[0], l.out_shape[1], P(cr["act_out"]), act_arg(conv_l), P(dzc), c,
                                         P(worker.grads) + cb.offset * 4 if cb else 0)
            rec[ci]["dz"], rec[ci]["dzT"] = dzc, dzcT
            continue
        if l.kind == "conv":
            ks = lay.by_name(l.kernel)
            r = rec[i]
            if i + 1 >= len(layers) or layers[i + 1].kind != "pool":
                # no pool after this conv: g_img is the gradient wrt its activation output (col2im of the next conv or the
                # flatten dgrad); dz = g * act'(a) and the bias gradient come from one kernel
                cb = lay.by_name(l.bias) if l.bias else None
                dzc = zeros(r["M"], ks.cols)
                plan.add_act_bwd_bias(P(g_img), ks.cols, r["M"], ks.cols, P(r["act_out"]), act_arg(l), P(dzc), ks.cols,
                                      P(worker.grads) + cb.offset * 4 if cb else 0)
                r["dz"], r["dzT"] = dzc, None
            kblocks = (r["M"] + 63) // 64
            tiles = ((r["K"] + 127) // 128) * max(1, (ks.cols + 63) // 64)
            if use_mn:
                # dW = patches^T . dz from the row-major im2col matrix and dz (no patches^T / dz^T are ever written)
                cw = dict(a=P(r["patches"]), lda=r["ldK"], b=P(r["dz"]), ldb=ks.cols, M=r["K"], N=ks.cols, K=r["M"], mn_major=1,
                          split_k=_split_k(tiles, kblocks), accumulate=1)
            else:
                cw = dict(a=P(r["patchesT"]), lda=r["ldM"], b=P(r["dzT"]), ldb=r["ldM"], M=r["K"], N=ks.cols, K=r["M"],
                          split_k=_split_k(tiles, kblocks), accumulate=1)
            if sharded:
                cw.update(worker.route_args(ks))          # red.add into the owners' mailboxes (appliers hand them back zeroed)
            else:
                cw.update(out_f32=P(worker.grads) + ks.offset * 4, ld_f32=ks.cols)
            wg = C.Gemm(cw)
            gemms.append(wg)
            r["wgrad"] = wg
            if wgrad_on_side(i):
                side(lambda wg=wg, i=i: plan.add_gemm(wg, f"wgrad{i}"))
            else:
                plan.add_gemm(wg, f"wgrad{i}")
            if i == first_trainable:
                break
            h, w, cin = r["in_shape"]
            dpatch = zeros(r["M"], r["ldK"])
            dg = C.Gemm(dict(a=P(r["dz"]), lda=ks.cols, b=P(wsrc) + ks.w_off * 2, ldb=ks.w_ld, M=r["M"], N=r["K"], K=ks.cols,
                             out_bf16=P(dpatch), ld_bf16=r["ldK"], a_evict_first=1))
            gemms.append(dg)
            plan.add_gemm(dg, f"dgrad{i}")
            g_img = zeros(B, h * w * cin)
            plan.add_col2im(P(dpatch), r["ldK"], B, h, w, cin, l.ksize[0], l.ksize[1], P(g_img), l.strides[0], l.strides[1], l.pads[0],
                            l.pads[2], l.out_shape[0], l.out_shape[1])
            continue
    if sharded and with_push:
        # forward the 1-D tail (bias gradients, all complete by now on the main branch) beside the last wgrad, so the post
        # after the join is a bare flag store: no store of its own to order, no system fence on the critical path
        plan.add_post_flags(worker._post_flags_args(loss_out, phase=1))
    for b in (2, 1)[:n_side[0]]:
        plan.join(b)
    if with_push:
        extra = dict(done_dev=P(done_dev)) if done_dev is not None else {}
        if sharded:
            plan.add_post_flags(dict(worker._post_flags_args(loss_out, phase=2), **extra))
        elif worker.served:
            plan.add_post(dict(worker._post_args(loss_out), **extra), P(worker.sync_push), 0)
        else:
            plan.add_push(dict(worker._push_args(loss_out), **extra), P(worker.sync_push), 0)
    keep.append(gemms)
    return BuiltPlan(plan, x_stage, y_stage, loss_out, None, keep, rec)
