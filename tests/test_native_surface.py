"""The Python surface of the native module (no GPU): every module function and every Plan method of ``_C``, by name
and pybind signature line (argument names, order and defaults), against the list below.  Each kernel is bound once in
csrc/runtime.cpp and exposed twice, as ``Plan.add_<op>`` and as a direct entry point; this pins both forms, including
the plan / direct name pairs that differ (add_mse / mse_loss, add_argmax / argmax_rows) and the conv kernels whose
direct form takes its stream before the defaulted geometry arguments."""
import inspect

import pytest

# pybind11 spells an integer parameter as this union; the lists below write it as `int`
_INT = "typing.SupportsInt | typing.SupportsIndex"


def _signature(name, obj):
    doc = getattr(obj, "__doc__", None) or ""
    line = doc.splitlines()[0] if doc else ""
    return line.replace(_INT, "int") if line.startswith(name + "(") else None


MODULE_FUNCTIONS = {
    "act_bwd_bias": (
        "act_bwd_bias(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: int, "
        "arg9: int) -> None"),
    "argmax_rows": "argmax_rows(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int) -> None",
    "cast_transpose": (
        "cast_transpose(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: "
        "int, arg9: int) -> None"),
    "col2im": (
        "col2im(dcols: int, ld_cols: int, n: int, h: int, w: int, c: int, kh: int, kw: int, din: int, stream: int, sh: "
        "int = 1, sw: int = 1, pad_top: int = 0, pad_left: int = 0, out_h: int = 0, out_w: int = 0) -> None"),
    "conv_first_fwd": (
        "conv_first_fwd(x: int, n: int, h: int, w: int, cin: int, kh: int, kw: int, cout: int, wT: int, ld_w: int, bias: "
        "int, act: int, pooled: int, argmax: int, stream: int, pad_top: int = 0, pad_left: int = 0, out_h: int = 0, "
        "out_w: int = 0) -> None"),
    "conv_first_wgrad": (
        "conv_first_wgrad(x: int, n: int, h: int, w: int, cin: int, kh: int, kw: int, cout: int, g_pool: int, pooled: "
        "int, argmax: int, act: int, dW: int, db: int, stream: int, pad_top: int = 0, pad_left: int = 0, out_h: int = 0, "
        "out_w: int = 0) -> None"),
    "device_count": "device_count() -> int",
    "enable_peer_access": "enable_peer_access(arg0: int) -> bool",
    "gemm_pick_bn": "gemm_pick_bn(arg0: int, arg1: int) -> int",
    "im2col": (
        "im2col(in: int, n: int, h: int, w: int, c: int, kh: int, kw: int, out: int, ld_out: int, outT: int, ld_t: int, "
        "stream: int, sh: int = 1, sw: int = 1, pad_top: int = 0, pad_left: int = 0, out_h: int = 0, out_w: int = 0) -> "
        "None"),
    "init_error_channel": "init_error_channel() -> None",
    "ipc_alloc": "ipc_alloc(arg0: int) -> int",
    "ipc_close_handle": "ipc_close_handle(arg0: int) -> None",
    "ipc_free": "ipc_free(arg0: int) -> None",
    "ipc_get_handle": "ipc_get_handle(arg0: int) -> bytes",
    "ipc_open_handle": "ipc_open_handle(arg0: str) -> int",
    "lock_op": "lock_op(arg0: int, arg1: int, arg2: int) -> None",
    "maxpool_bwd": (
        "maxpool_bwd(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: int, "
        "arg9: int, arg10: int, arg11: int, arg12: int, arg13: int) -> None"),
    "maxpool_fwd": (
        "maxpool_fwd(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: int, "
        "arg9: int) -> None"),
    "maxpool_gen_bwd": (
        "maxpool_gen_bwd(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: "
        "int, arg9: int, arg10: int, arg11: int, arg12: int, arg13: int, arg14: int, arg15: int, arg16: int, arg17: int, "
        "arg18: int, arg19: int) -> None"),
    "maxpool_gen_fwd": (
        "maxpool_gen_fwd(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: "
        "int, arg9: int, arg10: int, arg11: int, arg12: int, arg13: int, arg14: int, arg15: int) -> None"),
    "mc_add_device": "mc_add_device(arg0: int, arg1: int) -> None",
    "mc_bind": "mc_bind(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int) -> None",
    "mc_create": "mc_create(arg0: int, arg1: int) -> int",
    "mc_unbind": "mc_unbind(arg0: int, arg1: int, arg2: int, arg3: int) -> None",
    "memset_d8": "memset_d8(arg0: int, arg1: int, arg2: int) -> None",
    "mse_loss": (
        "mse_loss(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: int, "
        "arg9: int, arg10: int, arg11: int, arg12: int, arg13: int) -> None"),
    "pack_route": (
        "pack_route(arg0: int, arg1: collections.abc.Sequence[int], arg2: collections.abc.Sequence[int]) -> bytes"),
    "pack_ryw": "pack_ryw(arg0: int, arg1: collections.abc.Sequence[int], arg2: int, arg3: int, arg4: int) -> bytes",
    "pack_segs": "pack_segs(arg0: collections.abc.Sequence[collections.abc.Sequence[int]]) -> bytes",
    "post": "post(arg0: dict, arg1: int, arg2: int, arg3: int) -> None",
    "post_flags": "post_flags(arg0: dict, arg1: int) -> None",
    "pull": "pull(arg0: dict, arg1: int, arg2: int, arg3: int) -> None",
    "push": "push(arg0: dict, arg1: int, arg2: int, arg3: int) -> None",
    "read_error_code": "read_error_code() -> int",
    "read_host_error_code": "read_host_error_code() -> int",
    "set_pdl": "set_pdl(arg0: int) -> None",
    "sigmoid_xent": (
        "sigmoid_xent(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: int, "
        "arg9: int, arg10: int, arg11: int, arg12: int) -> None"),
    "softmax_xent": (
        "softmax_xent(arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: int, arg7: int, arg8: int, "
        "arg9: int, arg10: int, arg11: int, arg12: int) -> None"),
    "sync_pull": "sync_pull(arg0: dict, arg1: int) -> None",
    "trace_count": "trace_count() -> int",
    "trace_enable": "trace_enable(arg0: int, arg1: int) -> None",
    "vmm_create": "vmm_create(arg0: int, arg1: int) -> int",
    "vmm_export_fd": "vmm_export_fd(arg0: int) -> int",
    "vmm_granularity": "vmm_granularity(device: int, multicast: bool = False, n_devices: int = 1) -> int",
    "vmm_import_fd": "vmm_import_fd(arg0: int) -> int",
    "vmm_map": "vmm_map(arg0: int, arg1: int, arg2: collections.abc.Sequence[int]) -> int",
    "vmm_multicast_supported": "vmm_multicast_supported(arg0: int) -> bool",
    "vmm_release": "vmm_release(arg0: int) -> None",
    "vmm_unmap": "vmm_unmap(arg0: int, arg1: int) -> None",
}
PLAN_METHODS = {
    "__init__": "__init__(self: sparkflow_b200._C.Plan) -> None",
    "__len__": "__len__(self: sparkflow_b200._C.Plan) -> int",
    "add_act_bwd_bias": (
        "add_act_bwd_bias(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int,"
        " arg6: int, arg7: int, arg8: int) -> None"),
    "add_argmax": (
        "add_argmax(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int) -> None"),
    "add_cast_transpose": (
        "add_cast_transpose(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: "
        "int, arg6: int, arg7: int, arg8: int) -> None"),
    "add_col2im": (
        "add_col2im(self: sparkflow_b200._C.Plan, dcols: int, ld_cols: int, n: int, h: int, w: int, c: int, kh: int, kw: "
        "int, din: int, sh: int = 1, sw: int = 1, pad_top: int = 0, pad_left: int = 0, out_h: int = 0, out_w: int = 0) ->"
        " None"),
    "add_conv_first_fwd": (
        "add_conv_first_fwd(self: sparkflow_b200._C.Plan, x: int, n: int, h: int, w: int, cin: int, kh: int, kw: int, "
        "cout: int, wT: int, ld_w: int, bias: int, act: int, pooled: int, argmax: int, pad_top: int = 0, pad_left: int = "
        "0, out_h: int = 0, out_w: int = 0) -> None"),
    "add_conv_first_wgrad": (
        "add_conv_first_wgrad(self: sparkflow_b200._C.Plan, x: int, n: int, h: int, w: int, cin: int, kh: int, kw: int, "
        "cout: int, g_pool: int, pooled: int, argmax: int, act: int, dW: int, db: int, pad_top: int = 0, pad_left: int = "
        "0, out_h: int = 0, out_w: int = 0) -> None"),
    "add_gather_rows": (
        "add_gather_rows(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, "
        "arg6: int) -> None"),
    "add_gemm": "add_gemm(self: sparkflow_b200._C.Plan, gemm: sparkflow_b200._C.Gemm, name: str = 'gemm') -> None",
    "add_im2col": (
        "add_im2col(self: sparkflow_b200._C.Plan, in: int, n: int, h: int, w: int, c: int, kh: int, kw: int, out: int, "
        "ld_out: int, outT: int, ld_t: int, sh: int = 1, sw: int = 1, pad_top: int = 0, pad_left: int = 0, out_h: int = "
        "0, out_w: int = 0) -> None"),
    "add_maxpool_bwd": (
        "add_maxpool_bwd(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, "
        "arg6: int, arg7: int, arg8: int, arg9: int, arg10: int, arg11: int, arg12: int) -> None"),
    "add_maxpool_fwd": (
        "add_maxpool_fwd(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, "
        "arg6: int, arg7: int, arg8: int) -> None"),
    "add_maxpool_gen_bwd": (
        "add_maxpool_gen_bwd(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: "
        "int, arg6: int, arg7: int, arg8: int, arg9: int, arg10: int, arg11: int, arg12: int, arg13: int, arg14: int, "
        "arg15: int, arg16: int, arg17: int, arg18: int) -> None"),
    "add_maxpool_gen_fwd": (
        "add_maxpool_gen_fwd(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: "
        "int, arg6: int, arg7: int, arg8: int, arg9: int, arg10: int, arg11: int, arg12: int, arg13: int, arg14: int) -> "
        "None"),
    "add_mse": (
        "add_mse(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int, arg6: "
        "int, arg7: int, arg8: int, arg9: int, arg10: int, arg11: int, arg12: int) -> None"),
    "add_post": "add_post(self: sparkflow_b200._C.Plan, arg0: dict, arg1: int, arg2: int) -> None",
    "add_post_flags": "add_post_flags(self: sparkflow_b200._C.Plan, arg0: dict) -> None",
    "add_pull": "add_pull(self: sparkflow_b200._C.Plan, arg0: dict, arg1: int, arg2: int) -> None",
    "add_push": "add_push(self: sparkflow_b200._C.Plan, arg0: dict, arg1: int, arg2: int) -> None",
    "add_sigmoid_xent": (
        "add_sigmoid_xent(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int,"
        " arg6: int, arg7: int, arg8: int, arg9: int, arg10: int, arg11: int) -> None"),
    "add_softmax_xent": (
        "add_softmax_xent(self: sparkflow_b200._C.Plan, arg0: int, arg1: int, arg2: int, arg3: int, arg4: int, arg5: int,"
        " arg6: int, arg7: int, arg8: int, arg9: int, arg10: int, arg11: int) -> None"),
    "add_sync_pull": "add_sync_pull(self: sparkflow_b200._C.Plan, arg0: dict) -> None",
    "branch": "branch(self: sparkflow_b200._C.Plan, arg0: int) -> None",
    "capture": "capture(self: sparkflow_b200._C.Plan, arg0: int) -> None",
    "captured": "captured(self: sparkflow_b200._C.Plan) -> bool",
    "fork": "fork(self: sparkflow_b200._C.Plan, arg0: int) -> None",
    "graph_nodes": "graph_nodes(self: sparkflow_b200._C.Plan) -> int",
    "join": "join(self: sparkflow_b200._C.Plan, arg0: int) -> None",
    "names": "names(self: sparkflow_b200._C.Plan) -> list[str]",
    "replay": "replay(self: sparkflow_b200._C.Plan, arg0: int) -> None",
    "replay_n": "replay_n(self: sparkflow_b200._C.Plan, arg0: int, arg1: int) -> None",
    "run": "run(self: sparkflow_b200._C.Plan, arg0: int) -> None",
}


def _ext():
    from sparkflow_b200.ops import native

    return native.cuda_ext()


def test_module_functions_keep_their_names_and_signatures():
    C = _ext()
    got = {n: _signature(n, o) for n, o in sorted(vars(C).items()) if inspect.isbuiltin(o)}
    assert got == MODULE_FUNCTIONS


def test_plan_methods_keep_their_names_and_signatures():
    C = _ext()
    got = {n: s for n in sorted(vars(C.Plan)) if (s := _signature(n, getattr(C.Plan, n))) is not None}
    assert got == PLAN_METHODS


def test_pointer_lists_and_variable_rows_keep_their_checks():
    """Host-side checks raised before anything is launched: the device-address lists of push, post_flags and the applier
    are bounded by what their argument structs hold, a variable-table row has seven entries, and pack_segs writes each
    row as the SfTensorSeg layout the kernels read (zeroed padding)."""
    import re
    import struct

    C = _ext()
    push = dict(state=16, ctrl=16, grad=16, segs=16, tile_map=16, num_tiles=1)
    for extra, msg in ((dict(shadow_dst=[16] * 9), "push: at most 8 publish destinations"),
                       (dict(vec_pub=[16] * 3), "push: at most 2 vec_pub targets"),
                       (dict(vec_dst=[16] * 9), "push: at most 8 vec_dst targets"),
                       (dict(seg_rows=[[0, 1, 1, -1, 0, -1]]), "push: seg_rows entries are (offset, rows, cols, w_off, w_ld, wt_off, wt_ld)")):
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            C.push(dict(push, **extra), 0, 1, 0)
    flags = dict(n_shards=2, bounds=[0, 4, 8], grad=16, my_posted=16)
    for posted, mailbox in (([16], [16, 16]), ([16, 16], [16]), ([16] * 9, [16] * 9)):
        with pytest.raises(RuntimeError, match="post_flags: one posted word and one mailbox per shard"):
            C.post_flags(dict(flags, posted=posted, mailbox=mailbox), 0)
    applier_push = dict(state=16, ctrl=16, grad=0, applier=1, segs=16, tile_map=16, num_tiles=8)
    for shard, msg in ((dict(ack=[16] * 9), "applier: at most 8 ack words"), (dict(ack=[16, 0]), "applier: ack words must be non-null"),
                       (dict(ver_begin=[16], ver_end=[16, 16]), "applier: ver_begin / ver_end lists must match (<= 8)"),
                       (dict(ver_begin=[16] * 9, ver_end=[16] * 9), "applier: ver_begin / ver_end lists must match (<= 8)")):
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            C.Applier(applier_push, 16, 64, 16, 2, 16, 1e-4, 1, 1, 0, 0, 0, shard)

    with pytest.raises(RuntimeError, match=re.escape("pack_segs: (offset, rows, cols, w_off, w_ld, wt_off, wt_ld)")):
        C.pack_segs([[0, 1, 1, -1, 0, -1]])
    with pytest.raises(RuntimeError, match="pack_segs: w_ld / w_off must be multiples of 8"):
        C.pack_segs([[0, 4, 4, 8, 12, -1, 0]])
    rows = [[0, 300, 256, 0, 256, 76800, 304], [76800, 1, 256, -1, 0, -1, 0]]
    assert C.SEG_BYTES == struct.calcsize("<qiiqi4xqi4x")
    assert C.pack_segs(rows) == b"".join(struct.pack("<qiiqi4xqi4x", *r) for r in rows)
