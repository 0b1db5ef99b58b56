"""No-GPU checks on the built kernel library (`cuobjdump` on sparkflow_b200/_C.so): the hot kernels must not keep their
working set in local memory (round 2 found the optimizer tile code spilling its whole tile state because one fallback loop
indexed a register array with a runtime bound: 34 % of the push kernel's stall samples were `STL`), and the GEMMs must be
wgmma / TMA kernels."""
import re
import subprocess

import pytest

from kernel_usage import SO, gemm_instances, needs_binary_utils, res_usage

pytestmark = needs_binary_utils

# SfEpi (csrc/sf_api.h)
GENERIC, FWD, LOSS, DGRAD, WGRAD, SIGMOID_LOSS, SPARSE_LOSS = range(7)
# (BN, MN, EPI, EXT, PEN) of every one-CTA GEMM kernel instance (kGemmKernels, csrc/gemm_sm90.cu)
GEMM_INSTANCES = ({(bn, False, GENERIC, ext, pen) for bn in (32, 64, 128, 256) for ext, pen in ((False, False), (True, False), (False, True))}
                  | {(bn, True, GENERIC, False, pen) for bn in (64, 128) for pen in (False, True)}
                  | {(bn, False, epi, ext, False) for epi in (FWD, LOSS, DGRAD) for bn in (32, 64) for ext in (False, True)}
                  | {(bn, True, WGRAD, False, pen) for bn in (64, 128) for pen in (False, True)}
                  | {(bn, False, SIGMOID_LOSS, False, False) for bn in (32, 64)}
                  | {(32, False, SPARSE_LOSS, False, False)})


def test_hot_kernels_have_no_stack_frame():
    use = res_usage()
    hot = [k for k in use if re.match(r"sf::(push_kernel|applier_kernel|sf_gemm_kernel|sf_gemm_pair_kernel|sync_pull_kernel|post_flags_kernel|"
                                      r"im2col_vec8_kernel|col2im_vec8_kernel|cast_transpose_kernel|conv_first_wgrad_kernel<5, 5, 1>)", k)]
    assert len(hot) >= 40, sorted(use)[:10]
    spilled = {k: use[k] for k in hot if use[k][1] != 0}
    assert not spilled, f"kernels with a local-memory stack frame (REG, STACK): {spilled}"
    # occupancy contracts the plan builder relies on: the applier CTA (512 threads) must fit one SM's register file,
    # the push kernel must keep two CTAs per SM
    assert all(use[k][0] * 512 <= 65536 for k in use if k.startswith("sf::applier_kernel")), {k: v for k, v in use.items() if "applier" in k}
    assert all(use[k][0] * 256 * 2 <= 65536 for k in use if k.startswith("sf::push_kernel")), {k: v for k, v in use.items() if "push_kernel" in k}


def test_gemm_kernel_instances_are_wgmma_tma_kernels():
    fn = subprocess.run(["cuobjdump", "-sass", "-fun", "_ZN2sf14sf_gemm_kernelILi32ELb0ELi0ELb0ELb0EEEv14CUtensorMap_stS1_14SfGemmEpilogueiiii", SO],
                        stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
    if "Function" not in fn:
        pytest.skip("cuobjdump -fun did not find the mangled name (toolkit version)")
    for mnemonic in ("HGMMA", "WARPGROUP", "UTMALDG", "SYNCS"):
        assert mnemonic in fn, f"{mnemonic} missing from sf_gemm_kernel<32, false, 0, false, false>"
    assert "HMMA." not in fn                                  # no legacy mma.sync path


def test_gemm_kernel_instances_are_the_table():
    """The GEMM kernels in the library are exactly the instances of the table and the two pair instances, and none of
    them keeps a stack frame (the PEN instances included)."""
    use = res_usage()
    assert len(GEMM_INSTANCES) == 35
    found = gemm_instances(use)
    assert set(found) == GEMM_INSTANCES, (sorted(set(found) - GEMM_INSTANCES), sorted(GEMM_INSTANCES - set(found)))
    assert sorted(k for k in use if k.startswith("sf::sf_gemm_pair_kernel")) == ["sf::sf_gemm_pair_kernel<false>", "sf::sf_gemm_pair_kernel<true>"]
    gemms = {k: v for k, v in use.items() if k.startswith("sf::sf_gemm_")}
    assert len(gemms) == 37, sorted(gemms)
    spilled = {k: v for k, v in gemms.items() if v[1] != 0}
    assert not spilled, f"GEMM kernels with a local-memory stack frame (REG, STACK): {spilled}"
