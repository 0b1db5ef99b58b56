"""No-GPU checks on the built kernel library (`cuobjdump` on sparkflow_b200/_C.so): the hot kernels must not keep their
working set in local memory (round 2 found the optimizer tile code spilling its whole tile state because one fallback loop
indexed a register array with a runtime bound: 34 % of the push kernel's stall samples were `STL`), and the GEMMs must be
wgmma / TMA kernels."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "sparkflow_b200", "_C.so")
pytestmark = pytest.mark.skipif(not os.path.exists(SO) or shutil.which("cuobjdump") is None or shutil.which("c++filt") is None,
                                reason="needs the built extension and the CUDA binary utilities")


def _res_usage():
    txt = subprocess.run(["cuobjdump", "-res-usage", SO], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, check=True).stdout
    names = re.findall(r"Function (\S+):\n\s+REG:(\d+) STACK:(\d+)", txt)
    dem = subprocess.run(["c++filt"], input="\n".join(n for n, _, _ in names), stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()
    return {re.sub(r"\(.*", "", d).replace("void ", ""): (int(r), int(s)) for d, (_, r, s) in zip(dem, names)}


def test_hot_kernels_have_no_stack_frame():
    use = _res_usage()
    hot = [k for k in use if re.match(r"sf::(push_kernel|applier_kernel|sf_gemm_kernel|sf_gemm_pair_kernel|sync_pull_kernel|post_flags_kernel|"
                                      r"im2col_vec8_kernel|col2im_vec8_kernel|cast_transpose_kernel|conv_first_wgrad_kernel<5, 5, 1>)", k)]
    assert len(hot) >= 40, sorted(use)[:10]
    spilled = {k: use[k] for k in hot if use[k][1] != 0}
    assert not spilled, f"kernels with a local-memory stack frame (REG, STACK): {spilled}"
    # occupancy contracts the plan builder relies on: the applier CTA (512 threads) must fit one SM's register file,
    # the push kernel must keep two CTAs per SM
    assert all(use[k][0] * 512 <= 65536 for k in use if k.startswith("sf::applier_kernel")), {k: v for k, v in use.items() if "applier" in k}
    assert all(use[k][0] * 256 * 2 <= 65536 for k in use if k.startswith("sf::push_kernel")), {k: v for k, v in use.items() if "push_kernel" in k}


def test_gemm_kernels_are_wgmma_tma_kernels():
    fn = subprocess.run(["cuobjdump", "-sass", "-fun", "_ZN2sf14sf_gemm_kernelILi32ELb0EEEv14CUtensorMap_stS1_14SfGemmEpilogueiiii", SO],
                        stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
    if "Function" not in fn:
        pytest.skip("cuobjdump -fun did not find the mangled name (toolkit version)")
    for mnemonic in ("HGMMA", "WARPGROUP", "UTMALDG", "SYNCS"):
        assert mnemonic in fn, f"{mnemonic} missing from sf_gemm_kernel<32, false>"
    assert "HMMA." not in fn                                  # no legacy mma.sync path
