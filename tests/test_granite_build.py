"""Build checks of the kernels the Granite scales and the ragged classifier touched (csrc/decode_kernels.cuh, stream_matvec*.cuh,
decode_batch.cuh, prefill*.cuh) that need no GPU: every instantiation compiles for sm_90a without local-memory spills."""
import pytest

from test_batch_decode_build import _entries

CHANGED = [r"k_stream_matvec_q8ILi", r"k_stream_matvec_f16ILi", r"k_matvec_f16ILi", r"k_rmsnorm_quantILb",
           r"k_attentionILi(64|128)E", r"k_stream_matvec_q8_batch", r"k_rmsnorm_quant_batch", r"k_pf_embed", r"k_gemm_f16_wgmma"]


@pytest.mark.parametrize("pattern", CHANGED)
def test_scaled_kernels_do_not_spill(pattern):
    e = _entries(pattern)
    assert e, f"no instantiation matches {pattern}"
    for name, (stack, st, ld) in e.items():
        assert (st, ld) == (0, 0), f"{name}: spill stores / loads = {st} / {ld}"
