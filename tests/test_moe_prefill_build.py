"""Build checks of the MoE tensor-core prefill (B200_PREFILL_TENSOR_CORE_EXACT_MOE) that need no GPU: the header, the Python and
Java constants, the export and its wrapper, and the ptxas report build() writes next to the library."""
import inspect
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "include", "b200llama.h")
LOG = os.path.join(ROOT, "gpullama3.java_b200", "csrc", "ptxas.log")
JAVA = os.path.join(ROOT, "gpullama3.java_b200", "java", "B200MasterPlan.java")


def _entries(pattern):
    if not os.path.exists(LOG):
        pytest.skip("no ptxas report: the library was not built in this tree")
    lines = open(LOG).read().splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S*" + pattern + r"\S*)'", line)
        if m:
            props = next((x for x in lines[i + 1:i + 4] if "spill stores" in x), "")
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
            out[m.group(1)] = tuple(int(v) for v in s.groups()) if s else None
    return out


def test_header_defines_the_mode_and_the_hook():
    hdr = open(HDR).read()
    assert "#define B200_PREFILL_TENSOR_CORE_EXACT_MOE 4" in hdr
    assert "#define B200_PREFILL_TENSOR_CORE_EXACT 3" in hdr
    assert re.search(r"int b200_test_gemm_i8_experts\(int32_t mode, int32_t n_experts, const int32_t \*counts, int32_t n, int32_t k, "
                     r"const int8_t \*aq, const float \*as,\s+const void \*bq, const void \*bq2, float \*c, int8_t \*hq, float \*hs\);", hdr)


def test_python_and_java_constants(pkg):
    P = pkg.B200MasterPlan
    assert P.PREFILL_TENSOR_CORE_EXACT_MOE == 4 and P.PREFILL_TENSOR_CORE_EXACT == 3
    assert '"tensor_core_exact_moe": 4' in inspect.getsource(P.set_prefill_mode)
    assert "public static final int PREFILL_TENSOR_CORE_EXACT_MOE = 4;" in open(JAVA).read()


def test_export_and_wrapper_signatures(pkg):
    N = pkg.native
    assert "b200_test_gemm_i8_experts" in N.EXPORTS
    assert list(inspect.signature(N.test_gemm_i8_experts).parameters) == ["mode", "counts", "aq", "a_scales", "bq", "bq2", "c", "hq", "hs"]
    assert list(inspect.signature(N.NativePlan.moe_chunk_routing).parameters) == ["self", "rows"]
    assert list(inspect.signature(pkg.B200MasterPlan.moe_chunk_routing).parameters) == ["self", "rows"]


def test_new_kernels_are_built_without_spills():
    """The chunk router for both families, the grouping, the gather, the grouped GEMM for its two epilogues and the combine: no stack
    frame and no spills."""
    e = _entries(r"k_xp_")
    kinds = {re.search(r"k_xp_([a-z]+)", n).group(1) for n in e}
    assert {"route", "group", "gather", "gemm", "combine"} <= kinds, sorted(e)
    assert {re.search(r"ILb(\d)E", n).group(1) for n in e if "k_xp_route" in n} == {"0", "1"}
    assert {re.search(r"ILi(\d)E", n).group(1) for n in e if "k_xp_gemm" in n} == {"0", "2"}
    for name, v in e.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"


def test_counted_families_are_unchanged():
    """The build tests of the other paths count kernels by name: the new kernels add none to their families."""
    assert len(_entries(r"k_routed_")) == 3
    assert len(_entries(r"k_moe_")) == 3
    assert {re.search(r"ILi(\d)E", n).group(1) for n in _entries(r"_ZN2pg9k_gemm_i8ILi")} == {"0", "1", "2"}
    for name in _entries(r"k_xp_"):
        for sub in ("k_routed_", "k_moe_", "_batch", "k_i8_norm", "k_i8_rope_kv", "k_i8_attention", "k_pf_", "k_sample", "k_score_rows", "k_gemm_i8"):
            assert sub not in name, (name, sub)
