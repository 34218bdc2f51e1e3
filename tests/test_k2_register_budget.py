"""Register budget of the mapper kernels on sm_90a, from the compiler alone (no GPU needed).

The mapper kernels run 2 CTAs x 14 warps per SM (unc_abi.cu: K2_WARPS, K2_MIN_CTAS), which caps them at 72 registers.
They are bound by instruction count x latency, so spill code in the event loop costs throughput directly.  These tests
compile unc_abi.cu once (about a minute) and hold all five mapper kernels to the register cap, and k2_map, k2_map_ord
and k2_map_stream to a spill-store budget and a 21-hop history walk in phase B2 free of local-memory traffic.  The
exact-ties kernels have no spill budget: their extra code is the serial pdqsort over global memory.
"""
import os
import re
import shutil
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import spill_report  # noqa: E402

pytestmark = pytest.mark.skipif(shutil.which("nvcc") is None or shutil.which("nvdisasm") is None,
                                reason="needs nvcc and nvdisasm")

K2_THREADS = 14 * 32
CTAS_PER_SM = 2
SPILL_STORE_BUDGET = 320        # bytes per kernel (568-644 before the event loop stopped holding its workspace pointers)
DEFAULT_KERNELS = ("k2_map", "k2_map_ord", "k2_map_stream")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    cubin, text = spill_report.compile_cubin(str(tmp_path_factory.mktemp("k2_cubin")))
    return spill_report.ptxas_stats(text), spill_report.spill_lines(cubin)


@pytest.mark.parametrize("kernel", spill_report.KERNELS)
def test_registers_allow_two_ctas_of_14_warps(compiled, kernel):
    regs = compiled[0][kernel]["regs"]
    assert regs <= 72 and regs * K2_THREADS * CTAS_PER_SM <= 65536, regs


@pytest.mark.parametrize("kernel", DEFAULT_KERNELS)
def test_spill_store_budget(compiled, kernel):
    s = compiled[0][kernel]
    assert s["spill_st"] <= SPILL_STORE_BUDGET, s


def _b2_walk_lines():
    src = open(os.path.join(ROOT, "uncalled_b200", "csrc", "unc_k2v2.cuh")).read().split("\n")
    first = next(i for i, l in enumerate(src) if "21 parent hops back through the history ring" in l) + 1
    last = next(i for i in range(first, len(src)) if re.search(r"float oldC", src[i])) + 1
    return range(first, last + 1)


@pytest.mark.parametrize("kernel", DEFAULT_KERNELS)
def test_no_local_memory_in_b2_walk(compiled, kernel):
    lines = compiled[1][kernel]
    hits = {n: v for (f, n), v in lines.items() if f == "unc_k2v2.cuh" and n in _b2_walk_lines()}
    assert not hits, hits
