"""Build checks of the bit-exact tensor-core prefill that need no GPU: the ptxas report build() writes next to the library."""
import os
import re

import pytest

LOG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpullama3.java_b200", "csrc", "ptxas.log")
NEW = r"(_ZN2pg9k_gemm_i8ILi\dEE\S*|_Z\d+k_i8_(?:norm|rope_kv|attention)I\S+)"


def _entries():
    if not os.path.exists(LOG):
        pytest.skip("no ptxas report: the library was not built in this tree")
    lines = open(LOG).read().splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '" + NEW + "'", line)
        if m:
            props = next((x for x in lines[i + 1:i + 4] if "spill stores" in x), "")
            s = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
            out[m.group(1)] = tuple(int(v) for v in s.groups()) if s else None
    return out


def test_every_instantiation_is_built_without_spills():
    """The GEMM for its three epilogues, the norm with and without the embedding gather, and RoPE / KV and attention for every decode
    head size: no stack frame and no spills (the head-32 attention form included)."""
    e = _entries()
    gemm = {re.search(r"ILi(\d)E", n).group(1) for n in e if "k_gemm_i8" in n}
    assert gemm == {"0", "1", "2"}, sorted(gemm)
    for kind in ("rope_kv", "attention"):
        sizes = {int(re.search(r"ILi(\d+)E", n).group(1)) for n in e if f"k_i8_{kind}" in n}
        assert sizes == {32, 64, 96, 128, 256}, (kind, sorted(sizes))
    assert {re.search(r"ILb(\d)E", n).group(1) for n in e if "k_i8_norm" in n} == {"0", "1"}
    for name, v in e.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"


def test_new_kernel_names_stay_out_of_the_counted_families():
    """The batched-step build tests count kernels by name; none of the new ones may be counted with them."""
    for name in _entries():
        for sub in ("_batch", "k_attention_batch", "k_rmsnorm_quant_batch", "k_stream_matvec_q8", "k_stream_matvec_kq", "k_rope_kv_batch",
                    "k_attention_cached_rows", "k_argmax_batch", "k_batch_rows_next", "k_pf_", "k_attentionILi", "k_rmsnorm_quantILb",
                    "k_gemm_f16_wgmma"):
            assert sub not in name, (name, sub)
