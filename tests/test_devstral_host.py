"""Devstral 2 on the host (no GPU): model type detection and the generation loop, DevstralModelLoader.createConfiguration's keys and
defaults (DevstralModelLoader.java:45-71) and its YaRN branch (:76-110), the value_length refusal, the tokenizer refusal, and the C ABI's
Devstral creator and YaRN struct."""
import ctypes as C
import os

import numpy as np
import pytest


def _write(pkg, path, shape_name="tiny-devstral", quant=None, edit=None):
    s = pkg.synth
    sh = s.SHAPES[shape_name]
    quant = pkg.gguf.GGMLType.Q8_0 if quant is None else quant
    md = s.metadata_for(sh, quant, f"Devstral synthetic {shape_name}")
    if edit:
        edit(md)
    pkg.gguf.write_gguf(path, md, s.build_tensors(sh, quant, 1234, 0.0))
    return sh


def test_devstral_type_and_loop(pkg):
    assert pkg.loader.detect_model_type({"general.name": "Devstral-Small-2-24B-Instruct-2512"}) == "DEVSTRAL_2"
    assert pkg.engine.loop_for("DEVSTRAL_2") is pkg.engine.generate_tokens_llama
    assert pkg.loader.ARCH_DEVSTRAL == 6


def test_devstral_configuration_keys(pkg, tmp_path):
    path = str(tmp_path / "d.gguf")
    sh = _write(pkg, path)
    m = pkg.load_model(path, 64)
    c = m.configuration
    assert m.model_type == "DEVSTRAL_2" and c.arch == 6 and c.quantization == "Q8_0"
    assert m.gguf.metadata["general.architecture"] == "mistral3"
    assert (c.dim, c.hidden_dim, c.n_layers, c.n_heads, c.n_kv_heads, c.head_size, c.vocab_size) == (512, 1024, 2, 4, 2, 64, 512)
    assert c.q_dim == 256 != c.dim                                             # head size from key_length, not dim / heads
    assert c.yarn == pkg.loader.Yarn(4.0, 32.0, 1.0, 1.0, 256)
    assert c.context_length == 64
    assert pkg.load_model(path, 10 ** 5).configuration.context_length == sh.model_ctx  # finalContextLength: clamped to the model's
    assert pkg.load_model(path).configuration.context_length == sh.model_ctx
    plain = str(tmp_path / "p.gguf")
    _write(pkg, plain, "tiny-devstral-plain")
    assert pkg.load_model(plain).configuration.yarn is None


def test_devstral_configuration_defaults_and_floats(pkg, tmp_path):
    def edit(md):
        for k in ("mistral3.attention.layer_norm_rms_epsilon", "mistral3.rope.freq_base", "mistral3.vocab_size", "mistral3.attention.head_count_kv",
                  "mistral3.rope.scaling.yarn_log_multiplier", "mistral3.attention.value_length"):
            del md[k]
        md["mistral3.rope.scaling.factor"] = 0.1          # read as a Java float
        md["tokenizer.ggml.tokens"] = [f"t{i}" for i in range(300)]
    path = str(tmp_path / "d.gguf")
    _write(pkg, path, edit=edit)
    c = pkg.load_model(path).configuration
    assert (c.rms_norm_eps, c.rope_theta) == (float(np.float32(1e-5)), 10000.0)
    assert c.vocab_size == 300                                                 # the token list's length
    assert c.n_kv_heads == c.n_heads
    assert c.yarn.log_multiplier == 0.0 and c.yarn.factor == float(np.float32(0.1))


def test_devstral_scaling_types(pkg, tmp_path):
    def other(md):
        md["mistral3.rope.scaling.type"] = "linear"       # the reference builds the plain table for any type but "yarn"
    p1 = str(tmp_path / "l.gguf")
    _write(pkg, p1, edit=other)
    assert pkg.load_model(p1).configuration.yarn is None

    def missing(md):
        del md["mistral3.rope.scaling.yarn_beta_fast"]
    p2 = str(tmp_path / "m.gguf")
    _write(pkg, p2, edit=missing)
    with pytest.raises(KeyError):
        pkg.load_model(p2)


def test_devstral_value_length_refused(pkg, tmp_path):
    def edit(md):
        md["mistral3.attention.value_length"] = 128
    path = str(tmp_path / "v.gguf")
    _write(pkg, path, edit=edit)
    with pytest.raises(pkg.loader.UnsupportedModel, match="value_length"):
        pkg.load_model(path)


def test_devstral_tokenizer_refused(pkg, tmp_path):
    path = str(tmp_path / "t.gguf")
    _write(pkg, path)
    m = pkg.load_model(path)
    with pytest.raises(pkg.tokenizer.UnsupportedTokenizer):
        pkg.tokenizer.from_metadata(m.gguf.metadata, m.model_type)


def test_devstral_abi(pkg):
    N = pkg.native
    assert "b200_plan_create_devstral" in N.EXPORTS
    names = [n for n, _ in N.YarnConfig._fields_]
    assert names == ["factor", "beta_fast", "beta_slow", "log_multiplier", "original_context_length"]
    assert C.sizeof(N.YarnConfig) == 20
    for i, n in enumerate(names):
        assert getattr(N.YarnConfig, n).offset == 4 * i
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200llama.h")).read()
    assert "#define B200_ARCH_DEVSTRAL 6" in hdr and "int b200_plan_create_devstral(" in hdr and "} b200_yarn_config;" in hdr
    assert hasattr(N.lib(), "b200_plan_create_devstral")


def test_host_code_is_built_without_fp_contraction(pkg):
    """The RoPE tables are evaluated on the host with Java's roundings: the host compiler must not fuse a*b+c."""
    flags = pkg.build.NVCC_FLAGS
    assert "-ffp-contract=off" in flags and flags[flags.index("-ffp-contract=off") - 1] == "-Xcompiler"
