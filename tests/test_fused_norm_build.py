"""Build checks of the normalising stream kernels (k_stream_matvec_q8_norm, csrc/stream_matvec.cuh + norm_slots.cuh) that need no
GPU: both instantiations (STORE for QKV and lm_head, GATEUP) compile for sm_90a without local-memory spills."""
from test_batch_decode_build import _entries


def test_fused_norm_kernels_do_not_spill():
    e = _entries(r"k_stream_matvec_q8_norm")
    assert len(e) == 2, sorted(e)
    for name, (stack, st, ld) in e.items():
        assert (st, ld) == (0, 0), f"{name}: spill stores / loads = {st} / {ld}"
