"""Build checks of the prefill GEMM that need no GPU: the ptxas report build() writes next to the library."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpullama3.java_b200", "csrc", "ptxas.log")


def _gemm_entries():
    if not os.path.exists(LOG):
        pytest.skip("no ptxas report: the library was not built in this tree")
    lines = open(LOG).read().splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(_ZN2pg16k_gemm_f16_wgmma\S+)'", line)
        if m:
            props = next((x for x in lines[i + 1:i + 4] if "spill stores" in x), "")
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
            out[m.group(1)] = tuple(int(v) for v in s.groups()) if s else None
    return out


def test_w8a16_gemm_instantiations_do_not_spill():
    """Every W8A16 instantiation (template argument BSRC = 1), for the three epilogues and both ring depths, compiles without a
    stack frame or spills; so do the f16 ones."""
    entries = _gemm_entries()
    q8 = {n: v for n, v in entries.items() if re.match(r"_ZN2pg16k_gemm_f16_wgmmaILi\dELi\dELi1EE", n)}
    modes = {(re.search(r"ILi(\d)ELi(\d)E", n).groups()) for n in q8}
    assert modes == {(m, s) for m in "012" for s in "45"}, sorted(modes)
    for name, v in entries.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"
