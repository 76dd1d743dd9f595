"""Checks of resident K-quant weights that need no GPU: the resident stream kernels (k_stream_matvec_kq / _kq_norm, csrc/stream_matvec.cuh)
compile for sm_90a in every mode and format without local-memory spills, and the new calls are exported and wrapped."""
import inspect

from test_batch_decode_build import _entries


def test_resident_stream_kernels_do_not_spill():
    plain = _entries(r"k_stream_matvec_kqI")
    norm = _entries(r"k_stream_matvec_kq_norm")
    assert len(plain) == 9, sorted(plain)  # STORE / RESID / GATEUP x Q4_K / Q5_K / Q6_K
    assert len(norm) == 6, sorted(norm)    # STORE / GATEUP x Q4_K / Q5_K / Q6_K
    q8 = _entries(r"k_stream_matvec_q8ILi")
    q8_stack = max(stack for stack, _, _ in q8.values())
    for name, (stack, st, ld) in {**plain, **norm}.items():
        assert (st, ld) == (0, 0), f"{name}: spill stores / loads = {st} / {ld}"
        assert stack <= q8_stack, f"{name}: {stack}-byte stack frame, the Q8_0 form has {q8_stack}"


def test_weight_calls_are_exported_and_wrapped(pkg):
    n = pkg.native
    assert {"b200_weight_info", "b200_test_set_memory_budget"} <= set(n.EXPORTS)
    assert list(inspect.signature(n.NativePlan.weight_info).parameters) == ["self"]
    assert list(inspect.signature(pkg.B200MasterPlan.weight_info).parameters) == ["self"]
    assert list(inspect.signature(n.test_set_memory_budget).parameters) == ["n_bytes"]
