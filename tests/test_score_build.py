"""Build checks of token scoring (b200_score_tokens) that need no GPU: the per-row reduction k_score_rows (csrc/score.cuh) and the int8
GEMM's classifier epilogue (k_gemm_i8_logits, csrc/prefill_i8.cuh) compile for sm_90a without local-memory spills or stack frames,
and the entry point is exported and wrapped at every layer."""
import inspect
import os

from test_batch_decode_build import _entries

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_score_kernels_do_not_spill():
    e = _entries(r"k_score_rows|k_gemm_i8_logits")
    assert len(e) == 2, sorted(e)
    for name, v in e.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"


def test_score_entry_point_is_exported_and_wrapped(pkg):
    n = pkg.native
    assert "b200_score_tokens" in n.EXPORTS
    assert list(inspect.signature(n.NativePlan.score_tokens).parameters) == ["self", "tokens", "start_pos", "targets"]
    assert list(inspect.signature(pkg.B200MasterPlan.score_tokens).parameters) == ["self", "tokens", "start_pos", "targets"]
    assert list(inspect.signature(pkg.engine.score_sequence).parameters) == ["plan", "tokens", "start_pos"]
    hdr = open(os.path.join(ROOT, "include", "b200llama.h")).read()
    assert "int b200_score_tokens(b200_plan *plan, const int32_t *tokens, const int32_t *targets, int32_t n, int32_t start_pos" in hdr
    java = open(os.path.join(ROOT, "gpullama3.java_b200", "java", "B200MasterPlan.java")).read()
    assert 'fn("b200_score_tokens"' in java and "public void scoreTokens(" in java
