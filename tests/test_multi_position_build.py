"""The multi-position step's kernels compile for sm_90a without spills (the ptxas report build() writes).  Head-32 attention
spills a few bytes in every form, the existing k_attention_batch<32> included, so it is held to that form's size."""
from test_batch_decode_build import _entries


def test_multi_position_kernels_do_not_spill():
    e = _entries(r"k_rope_kv_batch|k_attention_cached_rows")
    assert len([n for n in e if "k_rope_kv_batch" in n]) == 5, sorted(e)
    assert len([n for n in e if "k_attention_cached_rows" in n]) == 5, sorted(e)
    for name, (stack, st, ld) in e.items():
        if "k_attention_cached_rowsILi32E" in name:
            assert stack <= 32 and st <= 32 and ld <= 32, f"{name}: stack / spill stores / loads = {stack} / {st} / {ld}"
        else:
            assert (stack, st, ld) == (0, 0, 0), f"{name}: stack / spill stores / loads = {stack} / {st} / {ld}"
