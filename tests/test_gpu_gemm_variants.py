"""Specialized GEMM epilogue variants: each computes exactly what the generic kernel computes for the same GEMM, the
dense training plans select them, and none of them keeps a stack frame."""
import re

import pytest
import torch

from sparkflow_b200.ops import native
from kernel_usage import gemm_instances, needs_binary_utils, res_usage
from sparkflow_b200.ops.layout import round_up

# SfEpi (csrc/sf_api.h)
GENERIC, FWD, LOSS, DGRAD, WGRAD = 0, 1, 2, 3, 4
RELU, SIGMOID = 1, 2


def _bf16(rows, cols, ld, g, scale=0.5, fn=None):
    x = torch.randn(rows, cols, device="cuda", generator=g) * scale
    if fn is not None:
        x = fn(x)
    out = torch.zeros(rows, ld, dtype=torch.bfloat16, device="cuda")
    out[:, :cols] = x.to(torch.bfloat16)
    return out


def _case(kind, M, N, K, act=0, aux_act=RELU, loss_mode=1, split_k=1, bias=True, colsum=True, seed=0):
    """Operands (shared by both runs) and a factory of fresh outputs for one GEMM of the given kind."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ins = {}
    if kind == WGRAD:                    # both operands MN-major: a [K, M], b [K, N]
        lda, ldb = round_up(M, 8), round_up(N, 8)
        ins["a"], ins["b"] = _bf16(K, M, lda, g), _bf16(K, N, ldb, g)
    else:
        lda = ldb = round_up(K, 8)
        ins["a"], ins["b"] = _bf16(M, K, lda, g), _bf16(N, K, ldb, g)
    ldn = round_up(N, 8)
    d = dict(a=native.ptr(ins["a"]), b=native.ptr(ins["b"]), M=M, N=N, K=K, lda=lda, ldb=ldb, act=act, split_k=split_k)
    if kind in (FWD, LOSS) and bias:
        ins["bias"] = torch.randn(N, device="cuda", generator=g)
        d["bias"] = native.ptr(ins["bias"])
    if kind == DGRAD:
        fn = torch.relu if aux_act == RELU else torch.sigmoid
        ins["aux"] = _bf16(M, N, ldn, g, scale=1.0, fn=fn)
        d.update(aux=native.ptr(ins["aux"]), ld_aux=ldn, aux_act=aux_act)
    if kind == LOSS:
        if loss_mode == 1:
            ins["target"] = torch.eye(N, device="cuda")[torch.randint(0, N, (M,), device="cuda", generator=g)]
        else:
            ins["target"] = torch.rand(M, N, device="cuda", generator=g)
        d.update(loss_mode=loss_mode, target=native.ptr(ins["target"]), ld_target=N)
    if kind == WGRAD:
        d["mn_major"] = 1

    def outputs():
        o = {}
        if kind == WGRAD:
            o["f32"] = torch.full((M, N), 0.25, device="cuda")
            dd = dict(out_f32=native.ptr(o["f32"]), ld_f32=N)
        else:
            o["bf16"] = torch.full((M, ldn), 3.0, dtype=torch.bfloat16, device="cuda")
            dd = dict(out_bf16=native.ptr(o["bf16"]), ld_bf16=ldn)
        if kind in (LOSS, DGRAD) and colsum:
            o["colsum"] = torch.zeros(N, device="cuda")
            dd["colsum"] = native.ptr(o["colsum"])
        if kind == LOSS:
            o["loss"] = torch.zeros(1, device="cuda")
            dd["loss"] = native.ptr(o["loss"])
        return o, dd

    return ins, d, outputs


def _run(C, d, dd, epi):
    gm = C.Gemm(dict(d, **dd, epi=epi))
    gm.launch(native.current_stream())
    torch.cuda.synchronize()
    assert C.read_error_code() == 0
    return gm


CASES = [
    # simple_dnn 784-256-256-10, batch 300
    ("dnn_fwd0", FWD, 300, 256, 784, dict(act=RELU)),
    ("dnn_fwd1", FWD, 300, 256, 256, dict(act=RELU)),
    ("dnn_fwd2_xent", LOSS, 300, 10, 256, dict(loss_mode=1)),
    ("dnn_dgrad2", DGRAD, 300, 256, 10, dict(aux_act=RELU)),
    ("dnn_dgrad1", DGRAD, 300, 256, 256, dict(aux_act=RELU)),
    ("dnn_wgrad0", WGRAD, 784, 256, 300, {}),
    ("dnn_wgrad2", WGRAD, 256, 10, 300, {}),
    # autoencoder 784-256-128-256-784 (sigmoid code and reconstruction, MSE)
    ("ae_code", FWD, 300, 128, 256, dict(act=SIGMOID)),
    ("ae_rec_mse", LOSS, 300, 784, 256, dict(act=SIGMOID, loss_mode=2)),
    ("ae_dgrad_code", DGRAD, 300, 128, 256, dict(aux_act=SIGMOID)),
    ("ae_wgrad_rec", WGRAD, 256, 784, 300, {}),
    # cnn: the second conv as a GEMM over im2col patches (BN 64, several waves), the dense head, the flatten dgrad
    # (no bias, no activation, no column sum) and the split-K conv weight gradient (atomic accumulate)
    ("cnn_conv2", FWD, 30000, 64, 288, dict(act=RELU)),
    ("cnn_head_xent", LOSS, 300, 10, 1600, dict(loss_mode=1)),
    ("cnn_flatten_dgrad", FWD, 300, 1600, 10, dict(bias=False)),
    ("cnn_wgrad_dense", WGRAD, 1600, 10, 300, {}),
    ("cnn_wgrad_conv2", WGRAD, 288, 64, 30000, dict(split_k=8)),
    # a dgrad without a bias below it (no column sum)
    ("dgrad_no_colsum", DGRAD, 300, 256, 256, dict(colsum=False)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,M,N,K,kw", CASES, ids=[c[0] for c in CASES])
def test_variant_matches_generic_kernel(name, kind, M, N, K, kw):
    C = native.cuda_ext()
    ins, d, outputs = _case(kind, M, N, K, **kw)
    o_auto, dd_auto = outputs()
    o_gen, dd_gen = outputs()
    g_auto = _run(C, d, dd_auto, -1)
    g_gen = _run(C, d, dd_gen, GENERIC)
    assert g_auto.epi == kind, (name, g_auto.epi)
    assert g_gen.epi == GENERIC
    assert g_auto.bn == g_gen.bn and g_auto.split_k == g_gen.split_k
    if "bf16" in o_auto:
        assert torch.isfinite(o_auto["bf16"].float()).all()
        assert torch.equal(o_auto["bf16"], o_gen["bf16"]), name
    if "f32" in o_auto:
        if g_auto.split_k > 1:       # atomic accumulation: the order of the K-split partial sums is not fixed
            torch.testing.assert_close(o_auto["f32"], o_gen["f32"], rtol=1e-5, atol=1e-4)
        else:
            assert torch.equal(o_auto["f32"], o_gen["f32"]), name
    for k in ("colsum", "loss"):         # atomic sums over row blocks
        if k in o_auto:
            torch.testing.assert_close(o_auto[k], o_gen[k], rtol=1e-5, atol=1e-5)
    if "loss" in o_auto:
        assert o_auto["loss"].item() > 0


@pytest.mark.gpu
def test_generic_kernel_keeps_the_features_no_variant_has():
    """Dropout, a transposed output and an fp32 output beside the bf16 one stay on the generic kernel."""
    C = native.cuda_ext()
    ins, d, outputs = _case(FWD, 300, 256, 256, act=RELU)
    o, dd = outputs()
    t = torch.zeros(256, 304, dtype=torch.bfloat16, device="cuda")
    f = torch.zeros(300, 256, device="cuda")
    for extra in (dict(drop_keep=0.5, drop_seed=7), dict(outT_bf16=native.ptr(t), ld_t=304), dict(out_f32=native.ptr(f), ld_f32=256)):
        assert _run(C, d, dict(dd, **extra), -1).epi == GENERIC, extra
    assert _run(C, d, dd, -1).epi == FWD


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["simple_dnn", "autoencoder"])
def test_dense_training_plan_selects_a_variant_for_every_gemm(model):
    from sparkflow_b200.graph.executor import GraphProgram
    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.models import zoo
    from sparkflow_b200.models.compiler import compile_graph
    from sparkflow_b200.ops.layout import ParamLayout
    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs

    label = "y:0" if model != "autoencoder" else None
    ir = GraphIR.from_metagraph(zoo.build(model))
    lp = compile_graph(ir, "x:0", label)
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    master = MasterState(lay, spec, torch.device("cuda:0"))
    master.load_weights(GraphProgram(ir).init_weights(seed=1))
    worker = DeviceWorker(ir, "x:0", label, spec, master, acquire_lock=True, shared=False)
    plan, _ = worker.build_plan(300, 0)
    gemms = [g for grp in worker._keep[-1] if isinstance(grp, list) for g in grp if hasattr(g, "epi")]
    n_dense = sum(1 for n in plan.names() if re.match(r"(fwd|dgrad|wgrad)\d", n))
    assert len(gemms) == n_dense >= 6, plan.names()
    assert all(g.epi != GENERIC for g in gemms), (plan.names(), [g.epi for g in gemms])
    master.close()


@needs_binary_utils
def test_epilogue_variant_instances_have_no_stack_frame():
    # the FWD / LOSS / DGRAD / WGRAD instances without the extended activations or the penalty
    variants = {k: v for k, v in gemm_instances(res_usage()).items() if FWD <= k[2] <= WGRAD and not k[3] and not k[4]}
    assert len(variants) == 8, sorted(variants)
    assert all(s == 0 for _, s in variants.values()), variants
