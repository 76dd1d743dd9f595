"""Build check of the controlled sampler that needs no GPU: k_sample_ctl (csrc/sampler.cuh) compiles for sm_90a without a stack
frame or local-memory spills, and every entry point the header declares for it is exported by the library."""
import ctypes

from test_batch_decode_build import _entries


def test_controlled_sampler_does_not_spill():
    e = _entries(r"k_sample_ctl")
    assert len(e) == 1, sorted(e)
    for name, v in e.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"


def test_entry_points_are_in_the_library(pkg):
    lib = pkg.native.lib()
    for name in ("b200_set_sampling_controls", "b200_set_sample_history", "b200_read_sample_counts", "b200_test_sample_controls"):
        assert isinstance(getattr(lib, name), ctypes._CFuncPtr), name
