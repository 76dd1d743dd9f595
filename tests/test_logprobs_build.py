"""Build checks of generated-token log-probabilities (b200_set_logprobs) that need no GPU: k_token_logprobs (csrc/logprobs.cuh)
compiles for sm_90a without local-memory spills or a stack frame, and the entry points are exported and wrapped at every layer."""
import inspect
import os

from test_batch_decode_build import _entries

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_logprobs_kernel_does_not_spill():
    e = _entries(r"k_token_logprobs")
    assert len(e) == 1, sorted(e)
    for name, v in e.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"


def test_logprobs_entry_points_are_exported_and_wrapped(pkg):
    n = pkg.native
    assert {"b200_set_logprobs", "b200_read_logprobs"} <= set(n.EXPORTS)
    for cls in (n.NativePlan, pkg.B200MasterPlan):
        assert list(inspect.signature(cls.set_logprobs).parameters) == ["self", "top_n"]
        assert list(inspect.signature(cls.last_logprobs).parameters) == ["self"]
    eng = pkg.engine
    for f in (eng.generate_tokens_batch, eng.generate_tokens_llama_batch_prefill, eng.generate_tokens_batch_prefill,
              eng.generate_tokens_lookahead, eng.generate_tokens_continuous):
        p = inspect.signature(f).parameters
        assert "logprobs" in p and p["logprobs"].default is None, f.__name__
    hdr = open(os.path.join(ROOT, "include", "b200llama.h")).read()
    assert "#define B200_MAX_TOP_LOGPROBS 20" in hdr
    assert "int b200_set_logprobs(b200_plan *plan, int32_t top_n);" in hdr
    assert "int b200_read_logprobs(b200_plan *plan, int32_t max_rows, int32_t *n_rows, double *chosen, int32_t *top_ids" in hdr
    java = open(os.path.join(ROOT, "gpullama3.java_b200", "java", "B200MasterPlan.java")).read()
    assert 'fn("b200_set_logprobs"' in java and 'fn("b200_read_logprobs"' in java
    assert "public void setLogprobs(" in java and "public Logprobs lastLogprobs(" in java
