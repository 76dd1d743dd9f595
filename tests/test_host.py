"""Host-side logic (no GPU): GGUF container, loader conventions, generation-loop conventions,
and that the C-ABI library loads and exports every symbol include/b200llama.h declares."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gguf_roundtrip(pkg, tmp_path):
    g = pkg.gguf
    rng = np.random.default_rng(0)
    a = rng.standard_normal(64 * 32).astype(np.float32)
    tensors = [("a.weight", g.GGMLType.F32, (64, 32), pkg.synth.encode(a, g.GGMLType.F32)),
               ("b.weight", g.GGMLType.Q8_0, (64, 32), pkg.synth.encode(a, g.GGMLType.Q8_0)),
               ("c.weight", g.GGMLType.F16, (7,), pkg.synth.encode(a[:7], g.GGMLType.F16))]
    md = {"general.architecture": "llama", "general.name": "x", "k.int": 5, "k.float": 1.5, "k.bool": True,
          "k.strs": ["a", "bc"], "k.ints": [1, 2, 3]}
    p = str(tmp_path / "t.gguf")
    g.write_gguf(p, md, tensors)
    f = g.GGUFFile(p)
    assert f.version == 3 and f.metadata["k.int"] == 5 and f.metadata["k.strs"] == ["a", "bc"] and f.metadata["k.ints"] == [1, 2, 3]
    assert f.metadata["k.float"] == 1.5 and f.metadata["k.bool"] is True
    assert f.tensor_data_offset % 32 == 0
    for name, tt, dims, raw in tensors:
        ti = f.tensor_infos[name]
        assert ti.dims == dims and ti.ggml_type == tt and ti.offset % 32 == 0
        assert np.array_equal(f.tensor_bytes(name), raw)
    assert f.tensor_infos["b.weight"].n_bytes == 64 * 32 // 32 * 34  # Q8_0: 34 B / 32 elems (GGMLType.java:13)


def test_gguf_rejects_bad_magic(pkg, tmp_path):
    p = tmp_path / "bad.gguf"
    p.write_bytes(b"NOPE" + b"\0" * 64)
    with pytest.raises(ValueError):
        pkg.gguf.GGUFFile(str(p))


def test_q8_quantizer_matches_oracle_c(pkg, orc):
    rng = np.random.default_rng(1)
    x = rng.standard_normal(32 * 50).astype(np.float32)
    x[:32] = 0
    a = pkg.synth.quantize_q8_0(x)
    b = np.empty(50 * 34, dtype=np.uint8)
    orc.lib().oracle_quantize_q8_0(x.ctypes.data, len(x), b.ctypes.data)
    assert np.array_equal(a, b)


def test_loader_conventions(pkg, make_model):
    Q = pkg.gguf.GGMLType.Q8_0
    m = make_model("tiny-llama", Q, 48)
    c = m.configuration
    assert (c.arch, c.dim, c.hidden_dim, c.n_layers, c.n_heads, c.n_kv_heads, c.head_size) == (0, 256, 512, 2, 4, 2, 64)
    assert c.context_length == 48 and c.quantization == "Q8_0" and c.rope_theta == 500000.0
    assert "output.weight" in m.tensors
    t = make_model("tiny-llama-tied", pkg.gguf.GGMLType.F16, 48)
    assert "output.weight" not in t.tensors and t.configuration.quantization == "FP16"
    q = make_model("tiny-qwen3", Q, 48)
    assert q.configuration.arch == 1 and q.configuration.head_size == 128 and q.configuration.q_dim == 512
    assert pkg.loader.detect_model_type({"general.name": "Mistral-7B"}) == "MISTRAL"
    assert pkg.loader.detect_model_type({"general.name": "Meta Llama 3"}) == "LLAMA_3"
    assert pkg.loader.detect_model_type({"general.name": "Qwen3 4B"}) == "QWEN_3"
    assert pkg.loader.detect_model_type({}) == "UNKNOWN"


def test_generation_loop_conventions(pkg):
    """Llama: BOS-seeded latest token at pos 0 then the prompt shifted by one
    (InferenceEngine.java:96-145).  Qwen3: prompt from pos 0 and one skipped position
    after the last prompt token (InferenceEngine.java:175-225)."""
    calls = []

    def fwd(tok, pos):
        calls.append((tok, pos))
        return 100 + pos

    out = pkg.engine.generate_tokens_llama(fwd, 7, 0, [7, 11, 12], [], 6, 64)
    assert calls == [(7, 0), (7, 1), (11, 2), (12, 3), (103, 4), (104, 5)]
    assert out == [103, 104, 105]
    calls.clear()
    out = pkg.engine.generate_tokens_qwen3(fwd, 0, 0, [11, 12, 13], [], 8, 64)
    assert calls == [(11, 0), (12, 1), (13, 2), (102, 4), (104, 5), (105, 6), (106, 7)]
    assert out == [102, 104, 105, 106, 107]
    calls.clear()
    out = pkg.engine.generate_tokens_llama(fwd, 7, 0, [7], [101], 16, 64)
    assert out == [101] and calls[-1] == (7, 1)  # stop token ends the loop, included in the output


def test_mistral_loads_for_the_forward_pass_only(pkg, tmp_path):
    """SURVEY 8(f) N4: a Mistral GGUF uses the Llama forward and weight slots (MistralModelLoader.java:92-113); its context is clamped
    to the model's (:45-46).  Its tokenizer family is NOT implemented and must be rejected up front (ADVICE r1), not mis-tokenised."""
    path = str(tmp_path / "mistral.gguf")
    pkg.synth.write_model(path, "tiny-llama", pkg.gguf.GGMLType.Q8_0, seed=3, display_name="Mistral-7B-Instruct synthetic")
    m = pkg.load_model(path, 10 ** 6)
    assert m.model_type == "MISTRAL" and m.configuration.arch == 0
    assert m.configuration.context_length == pkg.synth.SHAPES["tiny-llama"].model_ctx  # clamped, unlike Llama
    assert pkg.load_model(path, 48).configuration.context_length == 48
    with pytest.raises(pkg.tokenizer.UnsupportedTokenizer):
        pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)


def test_phi3_loads_with_fused_tensors(pkg, tmp_path):
    """SURVEY 8(f) N4: a Phi-3 GGUF (Phi3ModelLoader.java:51-113): head size = dim / heads, the requested context length is kept, the
    fused attn_qkv / ffn_up tensors are present instead of q/k/v/gate; its SentencePiece tokenizer is rejected up front."""
    G = pkg.gguf.GGMLType
    path = str(tmp_path / "phi3.gguf")
    sh = pkg.synth.write_model(path, "tiny-phi3", G.Q8_0, seed=4)
    m = pkg.load_model(path, 10 ** 5)
    c = m.configuration
    assert m.model_type == "PHI_3" and c.arch == 2 and c.head_size == sh.dim // sh.n_heads == 96
    assert c.context_length == 10 ** 5 and pkg.load_model(path, -1).configuration.context_length == sh.model_ctx
    qkv = m.tensors["blk.0.attn_qkv.weight"]
    assert tuple(qkv[1]) == (sh.dim, sh.q_dim + 2 * sh.kv_dim) and tuple(m.tensors["blk.1.ffn_up.weight"][1]) == (sh.dim, 2 * sh.hidden)
    assert "blk.0.attn_q.weight" not in m.tensors and "blk.0.ffn_gate.weight" not in m.tensors
    with pytest.raises(pkg.tokenizer.UnsupportedTokenizer):
        pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)


def test_batch_prefill_loop_conventions(pkg):
    """InferenceEngineWithBatchPrefillDecode.generateTokensGPULlama (:163-251): chunks are written at startPosition+chunkStart,
    clamped to the token budget, and decode starts at startPosition+N -- also for a continuation (startPosition > 0)."""
    class FakePlan:
        def __init__(self):
            self.prefill, self.decode = [], []

        def forward_batch_prefill(self, toks, start):
            self.prefill.append((list(toks), start))

        def forward_decode(self, tok, pos, logits=False):
            self.decode.append((tok, pos))
            return None, 1000 + pos

    fp = FakePlan()
    out = pkg.engine.generate_tokens_llama_batch_prefill(fp, 7, 10, [21, 22, 23, 24, 25], [], 20, 64, 2)
    assert fp.prefill == [([7, 21], 10), ([22, 23], 12), ([24], 14)]
    assert fp.decode[0] == (25, 15) and fp.decode[-1][1] == 19 and out == [1015, 1016, 1017, 1018, 1019]
    # prompt longer than the budget: the last chunk is truncated instead of overrunning the KV cache
    fp = FakePlan()
    out = pkg.engine.generate_tokens_llama_batch_prefill(fp, 7, 0, list(range(30, 40)), [], 5, 64, 4)
    assert fp.prefill == [([7, 30, 31, 32], 0), ([33], 4)] and out == [] and fp.decode == []
    with pytest.raises(IndexError):
        pkg.engine.generate_tokens_llama_batch_prefill(FakePlan(), 7, 0, [], [], 5, 64, 4)
    # equals the token-by-token loop on the same fake forward (which ignores history)
    calls = []
    ref = pkg.engine.generate_tokens_llama(lambda t, p: (calls.append((t, p)), 1000 + p)[1], 7, 10, [21, 22, 23, 24, 25], [], 20, 64)
    assert ref == [1015, 1016, 1017, 1018, 1019]


def test_abi_exports_every_declared_symbol(pkg):
    hdr = open(os.path.join(ROOT, "include", "b200llama.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations found"
    lib = ctypes.CDLL(pkg.native.LIB_PATH)
    for sym in declared:
        assert hasattr(lib, sym), f"{sym} declared in include/b200llama.h but not exported"
    assert set(pkg.native.EXPORTS) == declared
    lib.b200_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.b200_version()  # pure string getter; no compute call without a GPU


def test_native_struct_layout_matches_header(pkg):
    # b200_config: 9 int32, 2 float, 3 int32 = 56 bytes; b200_tensor: 2 pointers, 2 int32, 4 int64 = 56 bytes
    assert ctypes.sizeof(pkg.native.Config) == 56
    assert ctypes.sizeof(pkg.native.Tensor) == 56


def test_product_never_imports_oracle():
    """The product path must not import, link or load anything under oracle/."""
    pat = re.compile(r"(^\s*(import|from)\s+\S*oracle)|liboracle|oracle\.py|oracle\.c|import_oracle|dlopen.*oracle", re.M)
    pkgdir = os.path.join(ROOT, "gpullama3.java_b200")
    for dirpath, _, files in os.walk(pkgdir):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".java")):
                src = open(os.path.join(dirpath, fn), errors="replace").read()
                assert not pat.search(src), f"{fn}: product code references the oracle"
