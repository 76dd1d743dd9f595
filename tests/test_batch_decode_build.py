"""Build checks of the batched decode kernels (csrc/decode_batch.cuh) that need no GPU: the ptxas report build() writes next to the
library."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpullama3.java_b200", "csrc", "ptxas.log")


def _entries(pattern):
    if not os.path.exists(LOG):
        pytest.skip("no ptxas report: the library was not built in this tree")
    lines = open(LOG).read().splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m and re.search(pattern, m.group(1)):
            props = next((x for x in lines[i + 1:i + 4] if "spill stores" in x), "")
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
            out[m.group(1)] = tuple(int(v) for v in s.groups())
    return out


def test_batched_kernels_do_not_spill():
    """The three batched stream forms, the two batched norms, the argmax and the attention at head sizes 64 / 96 / 128 / 256 compile
    without local-memory spills.  The head-32 attention is the exception: its single-row form (k_attention<32>) spills as well."""
    e = _entries(r"_batch")
    assert len([n for n in e if "k_stream_matvec_q8_batch" in n]) == 3
    assert len([n for n in e if "k_rmsnorm_quant_batch" in n]) == 2
    assert len([n for n in e if "k_attention_batch" in n]) == 5
    assert len([n for n in e if "k_argmax_batch" in n]) == 1
    for name, (stack, st, ld) in e.items():
        if "k_attention_batchILi32E" in name:
            continue
        assert (st, ld) == (0, 0), f"{name}: spill stores / loads = {st} / {ld}"
    for name in [n for n in e if "k_stream_matvec_q8_batch" in n or "k_argmax_batch" in n]:
        assert e[name][0] == 0, f"{name}: stack frame {e[name][0]} bytes"
