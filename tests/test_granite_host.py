"""Granite 3.x on the host (no GPU): model type detection and the generation loop, GraniteLoader.createConfiguration's keys and defaults
(GraniteLoader.java:48-92), a synthetic GGUF round trip, the tokenizer refusal, and the C ABI's Granite creator and struct."""
import ctypes as C
import os

import numpy as np
import pytest


def _write(pkg, path, shape_name="tiny-granite", quant=None, edit=None):
    s = pkg.synth
    sh = s.SHAPES[shape_name]
    quant = pkg.gguf.GGMLType.Q8_0 if quant is None else quant
    md = s.metadata_for(sh, quant, f"Granite synthetic {shape_name}")
    if edit:
        edit(md)
    pkg.gguf.write_gguf(path, md, s.build_tensors(sh, quant, 1234, 0.0))
    return sh


def test_granite_type_and_loop(pkg):
    assert pkg.loader.detect_model_type({"general.name": "granite-3.1-8b-instruct"}) == "GRANITE"
    assert pkg.loader.detect_model_type({"general.name": "Granite 3.3 2B Instruct"}) == "GRANITE"
    assert pkg.engine.loop_for("GRANITE") is pkg.engine.generate_tokens_llama
    assert pkg.loader.ARCH_GRANITE == 5


def test_granite_configuration_keys(pkg, tmp_path):
    path = str(tmp_path / "g.gguf")
    sh = _write(pkg, path)
    m = pkg.load_model(path, 64)
    c = m.configuration
    assert m.model_type == "GRANITE" and c.arch == 5 and c.quantization == "Q8_0"
    assert (c.dim, c.hidden_dim, c.n_layers, c.n_heads, c.n_kv_heads, c.head_size, c.vocab_size) == (256, 512, 2, 4, 4, 64, 515)
    s = pkg.synth.GRANITE_SCALES
    assert (c.embedding_scale, c.residual_scale, c.attention_scale, c.logit_scale) == tuple(float(np.float32(s[k])) for k in
                                                                                              ("embedding_scale", "residual_scale", "attention_scale", "logit_scale"))
    assert c.context_length == 64                                             # the requested length
    assert pkg.load_model(path, 10 ** 5).configuration.context_length == 10 ** 5  # withContextLength keeps any length >= 0
    assert pkg.load_model(path).configuration.context_length == sh.model_ctx
    assert "output.weight" not in m.tensors                                    # tied classifier


def test_granite_configuration_defaults(pkg, tmp_path):
    def strip(md):
        for k in ("granite.embedding_scale", "granite.residual_scale", "granite.attention.scale", "granite.logit_scale",
                  "granite.attention.layer_norm_rms_epsilon", "granite.rope.freq_base", "granite.vocab_size", "granite.attention.head_count_kv"):
            del md[k]
    path = str(tmp_path / "d.gguf")
    _write(pkg, path, edit=strip)
    c = pkg.load_model(path).configuration
    assert (c.embedding_scale, c.residual_scale, c.attention_scale, c.logit_scale) == (12.0, float(np.float32(0.22)), 0.0078125, 16.0)
    assert (c.rms_norm_eps, c.rope_theta) == (float(np.float32(1e-5)), 10000.0)
    assert c.vocab_size == 515                                                 # the token list's length
    assert c.n_kv_heads == c.n_heads                                           # no GQA without the key


def test_granite_head_count_kv_forms(pkg, tmp_path):
    def arr(md):
        md["granite.attention.head_count_kv"] = [2, 2]
    p1 = str(tmp_path / "a.gguf")
    _write(pkg, p1, edit=arr)
    assert pkg.load_model(p1).configuration.n_kv_heads == 2

    def ragged(md):
        md["granite.attention.head_count_kv"] = [2, 4]
    p2 = str(tmp_path / "r.gguf")
    _write(pkg, p2, edit=ragged)
    with pytest.raises(pkg.loader.UnsupportedModel, match="varies across layers"):
        pkg.load_model(p2)


def test_granite_gguf_round_trip(pkg, tmp_path):
    path = str(tmp_path / "rt.gguf")
    sh = _write(pkg, path, "tiny-granite-gqa", pkg.gguf.GGMLType.F16)
    m = pkg.load_model(path, 32)
    assert m.configuration.quantization == "FP16" and m.configuration.n_kv_heads == 2 and m.configuration.head_size == 128
    want = {n: d for n, _, d, _ in pkg.synth.build_tensors(sh, pkg.gguf.GGMLType.F16, 1234, 0.0)}
    assert set(m.tensors) == set(want)
    for n, d in want.items():
        assert tuple(int(x) for x in m.tensors[n][1]) == tuple(d)


def test_granite_tokenizer_refused(pkg, tmp_path):
    path = str(tmp_path / "t.gguf")
    _write(pkg, path)
    m = pkg.load_model(path)
    with pytest.raises(pkg.tokenizer.UnsupportedTokenizer):
        pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)


def test_granite_abi(pkg):
    N = pkg.native
    assert "b200_plan_create_granite" in N.EXPORTS
    fields = [(n, t) for n, t in N.GraniteConfig._fields_]
    assert [n for n, _ in fields] == ["embedding_scale", "residual_scale", "attention_scale", "logit_scale"]
    assert all(t is C.c_float for _, t in fields) and C.sizeof(N.GraniteConfig) == 16
    for i, (n, _) in enumerate(fields):
        assert getattr(N.GraniteConfig, n).offset == 4 * i
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200llama.h")).read()
    assert "#define B200_ARCH_GRANITE 5" in hdr and "int b200_plan_create_granite(" in hdr
    lib = N.lib()
    assert hasattr(lib, "b200_plan_create_granite")
