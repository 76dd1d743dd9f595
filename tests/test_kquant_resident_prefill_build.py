"""Checks of the resident plan's bit-exact tensor-core prefill that need no GPU: the expansion kernel k_kq_tiles_to_q8
(csrc/stream_matvec.cuh) compiles for sm_90a in every K-quant format without local-memory spills, and its test hook is exported and
wrapped."""
import inspect

from test_batch_decode_build import _entries


def test_expansion_kernels_do_not_spill():
    e = _entries(r"k_kq_tiles_to_q8")
    assert len(e) == 3, sorted(e)  # Q4_K / Q5_K / Q6_K
    for fmt in (12, 13, 14):
        assert any(f"k_kq_tiles_to_q8ILi{fmt}E" in n for n in e), (fmt, sorted(e))
    for name, v in e.items():
        assert v == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {v}"


def test_expansion_hook_is_exported_and_wrapped(pkg):
    n = pkg.native
    assert "b200_test_kq_tiles_to_q8" in n.EXPORTS
    assert list(inspect.signature(n.test_kq_tiles_to_q8).parameters) == ["ggml_type", "rows", "cols", "raw"]


def test_q8_tile_bytes_is_the_layout_arithmetic(pkg):
    """4-row groups x segments x units: 4096 columns in 2 segments of 2048 (2176-byte units), Qwen3-4B's 9728 in 4 of 2432 (2584
    bytes padded to 2592), a 6-row matrix in two groups."""
    q = pkg.native.q8_tile_bytes
    assert q(4, 4096) == 4 * 2 * 2176
    assert q(4, 9728) == 4 * 4 * 2592
    assert q(6, 256) == 8 * 272
