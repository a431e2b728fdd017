"""Static checks on the SASS of the built library (cuobjdump; no GPU needed).

  * the tensor-core / TMA kernels really are Hopper-native: warpgroup MMA (HGMMA) fed by TMA tensor loads (UTMALDG) in every
    GEMM variant, both fused sampler kernels and the head_dim-80 attention core, no mma.sync (HMMA) among them;
  * no `ELECT ... BRA.U.ANY` uniformisation loop around a single-thread instruction: the single-thread regions are entered through
    elect.sync (ptx::elect_one), see DESIGN.md section 3 -- with `lane == 0` nvcc wraps every TMA issue in such a loop.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "paella_b200", "libpaella_b200.so")


@pytest.fixture(scope="module")
def census():
    if shutil.which("cuobjdump") is None or not os.path.exists(SO):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    fn, counts = None, collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts[fn] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and fn:
            counts[fn][m.group(1).split(".")[0]] += 1
            if m.group(1).startswith("BRA.U.ANY"):
                counts[fn]["BRA.U.ANY"] += 1
    return counts


def _kernels(census, pattern):
    return {k: v for k, v in census.items() if re.search(pattern, k)}


# the tensor-core kernels, one parameter per family of template instances (mangled names:
# gemm_f16_kernel<BLOCK_N, MODE, AMODE> = gemm_f16_kernelILi<BLOCK_N>ELi<MODE>ELi<AMODE>E)
WGMMA_VARIANTS = [
    pytest.param(r"gemm_f16_kernelILi64E", id="gemm_f16_kernel_bn64"),
    pytest.param(r"gemm_f16_kernelILi128E", id="gemm_f16_kernel_bn128"),
    pytest.param(r"gemm_f16_kernelILi256E", id="gemm_f16_kernel_bn256"),
    pytest.param(r"gemm_f16_kernelILi\d+ELi\d+ELi1E", id="gemm_f16_kernel_conv_k4s2"),
    pytest.param(r"gemm_f16_kernelILi\d+ELi\d+ELi2E", id="gemm_f16_kernel_convT_k4s2"),
    pytest.param(r"fused_sampler_kernel", id="fused_sampler_kernel"),
    pytest.param(r"fused_sampler_shared_kernel", id="fused_sampler_shared_kernel"),
    pytest.param(r"attention_wgmma_kernel", id="attention_wgmma_kernel"),
]


@pytest.mark.parametrize("needle", WGMMA_VARIANTS)
def test_tensor_core_kernels_are_wgmma_and_tma(census, needle):
    ks = _kernels(census, needle)
    assert ks, f"no kernel matching {needle} in the library"
    for name, c in ks.items():
        assert c["HGMMA"] > 0 and c["UTMALDG"] > 0, (name, dict(c))
        assert c["HMMA"] == 0, f"{name}: mma.sync instructions in a wgmma kernel"


def test_attention_fallback_is_the_only_mma_sync_kernel(census):
    hmma = [k for k, c in census.items() if c["HMMA"] > 0]
    assert hmma and all("attention_kernel" in k for k in hmma), hmma


@pytest.mark.parametrize("needle", ["gemm_f16_kernel", "fused_sampler"] + WGMMA_VARIANTS)
def test_single_thread_regions_have_no_uniformisation_loops(census, needle):
    ks = _kernels(census, needle)
    assert ks, f"no kernel matching {needle} in the library"
    for name, c in ks.items():
        # a handful remain around mbarrier arrivals guarded by `lane == 0`; none may sit on an MMA or TMA issue path:
        # far fewer loops than tensor-core + TMA instructions
        assert c["BRA.U.ANY"] <= 2, (name, c["BRA.U.ANY"], c["HGMMA"], c["UTMALDG"])
