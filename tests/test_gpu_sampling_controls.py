"""GPU tests of the sampling controls (b200_set_sampling_controls, k_sample_ctl in csrc/sampler.cuh).  Bar: the kernel's id,
diagnostics, modified row and counts equal the numpy restatement (sampling_controls_oracle) and the oracle sampler bit for bit;
neutral controls give today's ids; every calling path equals a host loop of forward_decode(logits) -> restatement -> oracle choice
with a host-tracked history, and the device counts equal that history at the end."""
import numpy as np
import pytest

import sampling_controls_oracle as sco
from test_gpu_continuous import ARRIVALS, _requests
from test_gpu_kquant_resident import _model as _kquant_model, _resident_plan

pytestmark = pytest.mark.gpu

K = 10  # generated tokens per sequence


def _controls(pkg, **kw):
    return pkg.sampler.SamplingControls(**kw)


def _menu(pkg, row):
    """Every control alone, a -100 bias on the argmax, and all together."""
    S = lambda **kw: _controls(pkg, **kw)  # noqa: E731
    am = int(np.argmax(row))
    return {"top_k": S(top_k=40), "top_k_1": S(top_k=1), "min_p": S(min_p=0.05), "min_p_1": S(min_p=1.0), "rep": S(repetition_penalty=1.3),
            "rep_below_1": S(repetition_penalty=0.8), "freq": S(frequency_penalty=0.02), "pres": S(presence_penalty=0.7),
            "bias": S(logit_bias={am: -100.0}), "all": S(top_k=50, min_p=0.02, repetition_penalty=1.2, frequency_penalty=0.01,
                                                          presence_penalty=0.3, logit_bias={am: -100.0, 3: 1.5, len(row) - 1: -0.25})}


def _rows(V, rng):
    r = {"random": (rng.standard_normal(V) * 3).astype(np.float32)}
    t = np.round(rng.standard_normal(V) * 2).astype(np.float32)  # thousands tied at every value: ties straddle v_k
    r["ties"] = t
    z = (rng.standard_normal(V) - 1.0).astype(np.float32)
    z[::7] = 0.0  # negative and zero logits under the repetition penalty
    r["negative_zero"] = z
    return r


def _counts(V, rng):
    c = (rng.random(V) < 0.01) * rng.integers(1, 4, V)
    c[rng.integers(0, V, 5)] = [1000, 2500, 4000, 7, 3000]  # counts in the thousands
    return c.astype(np.int32)


@pytest.mark.parametrize("V", [128256, 151936, 49155, 512])
def test_kernel_matches_the_oracle(pkg, orc, V):
    n = pkg.native
    rng = np.random.default_rng(V)
    for rname, row in _rows(V, rng).items():
        counts = _counts(V, rng)
        for cname, c in _menu(pkg, row).items():
            want_row = sco.modify(row, counts, c.top_k, c.min_p, c.repetition_penalty, c.frequency_penalty, c.presence_penalty, c.logit_bias)
            for temp, topp in ((0.0, 0.0), (0.9, 0.0), (0.9, 0.9)):
                u = float(np.float32(rng.random()))
                tok, info, got_row, got_counts = n.test_sample_controls(row, counts, c, temp, topp, u)
                where = (rname, cname, temp, topp)
                assert np.array_equal(got_row.view(np.uint32), want_row.view(np.uint32)), where
                want = orc.argmax(want_row) if temp == 0.0 else orc.sample(want_row, temp, topp, u)
                assert tok == want, where
                want_counts = counts.copy()
                want_counts[tok] += 1
                assert np.array_equal(got_counts, want_counts), where
                if temp == 0.0:
                    assert info == [0, 0, 0, 0], where
                else:  # the unchanged sampler on the modified row: the same id and diagnostics
                    assert (tok, info) == n.test_sample(want_row, temp, topp, u)[:2], where


@pytest.mark.parametrize("V", [128256, 512])
def test_neutral_controls_change_nothing(pkg, orc, V):
    n = pkg.native
    rng = np.random.default_rng(7)
    neutral = _controls(pkg)
    for _ in range(4):
        row = np.round(rng.standard_normal(V) * 3, 1).astype(np.float32)
        counts = _counts(V, rng)
        for temp, topp in ((0.0, 0.0), (0.7, 0.0), (1.1, 0.9)):
            u = float(np.float32(rng.random()))
            tok, info, got_row, _ = n.test_sample_controls(row, counts, neutral, temp, topp, u)
            assert np.array_equal(got_row.view(np.uint32), row.view(np.uint32))
            if temp == 0.0:
                assert tok == orc.argmax(row)
            else:
                assert (tok, info) == n.test_sample(row, temp, topp, u)[:2]


# ---- every calling path against a host loop ----------------------------------------------------------------------------------------

def _modes(pkg, plan):
    out = []
    for mode in ("graph", "persistent"):
        try:
            plan.set_decode_mode(mode)
            out.append(mode)
        except pkg.native.B200Error:
            pass
    return out


class _Host:
    """One sequence's host loop: forward_decode's raw logits, the restatement, the oracle's choice, a host-tracked history."""

    def __init__(self, pkg, orc, vocab, controls, temp, topp, seed, history=()):
        self.orc, self.controls, self.temp, self.topp = orc, controls, temp, topp
        self.rng = pkg.sampler.L32X64MixRandom(seed) if temp else None
        self.counts = np.zeros(vocab, np.int64)
        for t in history:
            self.counts[t] += 1

    def choose(self, logits):
        u = self.rng.next_float1() if self.temp else 0.0
        if self.controls is None:
            return self.orc.argmax(logits) if self.temp == 0.0 else self.orc.sample(logits, self.temp, self.topp, u)
        return sco.step(self.orc, logits, self.counts, self.controls, self.temp, self.topp, u)[0]


def _host_chain(plan, host, first, n=K):
    plan.kv_reset()
    toks = [first]
    for p in range(n):
        lg, _ = plan.forward_decode(toks[-1], p)
        toks.append(host.choose(lg))
    return toks[1:]


SEQ = [dict(temp=0.0, topp=0.0), dict(temp=0.9, topp=0.0), dict(temp=1.0, topp=0.9)]


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_single_sequence_path(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, ctx=64, seed=21)
    V = m.configuration.vocab_size
    c = _controls(pkg, top_k=8, min_p=0.01, repetition_penalty=1.5, frequency_penalty=0.2, presence_penalty=0.5, logit_bias={5: 2.0, 6: -100.0})
    hist = [5, 5, 9, 1]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        for mode in _modes(pkg, plan):
            plan.set_decode_mode(mode)
            for s in SEQ:
                smp = pkg.sampler.Sampler(V, s["temp"], s["topp"], 77, controls=c, history=hist)
                plan.kv_reset()
                toks = [1]
                for p in range(K):
                    toks.append(smp.sample_token(plan, toks[-1], p))
                dev_counts = plan.sample_counts(-1)
                host = _Host(pkg, orc, V, c, s["temp"], s["topp"], 77, hist)
                assert toks[1:] == _host_chain(plan, host, 1), (mode, s)
                assert np.array_equal(dev_counts, host.counts), (mode, s)
    finally:
        plan.free()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_batch_path_with_controls_per_slot(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, ctx=64, seed=22)
    V = m.configuration.vocab_size
    S = lambda **kw: _controls(pkg, **kw)  # noqa: E731
    per_slot = [S(top_k=4), None, S(repetition_penalty=1.4, presence_penalty=0.2), S(min_p=0.2, logit_bias={2: 3.0}), None,
                S(frequency_penalty=0.3, top_k=16), S(logit_bias={7: -100.0}), S(top_k=1)]
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        R = min(8, plan.decode_multi_rows())
        assert R >= 2
        for mode in _modes(pkg, plan):
            plan.set_decode_mode(mode)
            plan.set_decode_slots(R)
            for i in range(R):
                plan.set_sampling_controls(i, per_slot[i])
            hosts = [_Host(pkg, orc, V, per_slot[i], **{k: v for k, v in SEQ[i % 3].items()}, seed=300 + i) for i in range(R)]
            dev_rng = [pkg.sampler.L32X64MixRandom(300 + i) if SEQ[i % 3]["temp"] else None for i in range(R)]
            toks = [[1 + i] for i in range(R)]
            for p in range(K):
                smp = [(SEQ[i % 3]["temp"], SEQ[i % 3]["topp"], dev_rng[i].next_float1() if dev_rng[i] else 0.0) for i in range(R)]
                ids, _ = plan.forward_decode_batch(list(range(R)), [t[-1] for t in toks], [p] * R, smp)
                for i in range(R):
                    toks[i].append(int(ids[i]))
            dev_counts = [plan.sample_counts(i) for i in range(R) if per_slot[i] is not None]
            want = [_host_chain(plan, hosts[i], 1 + i) for i in range(R)]
            assert [t[1:] for t in toks] == want, mode
            assert all(np.array_equal(d, h.counts) for d, h in zip(dev_counts, [hosts[i] for i in range(R) if per_slot[i] is not None])), mode
            # without sampling the batch is the raw model: greedy argmax, controls and counts untouched
            plan.slot_reset(0)
            before = plan.sample_counts(0)
            ids, lg = plan.forward_decode_batch([0], [1], [0], None, logits=True)
            assert ids[0] == orc.argmax(lg[0]) and np.array_equal(plan.sample_counts(0), before)
            plan.set_decode_slots(0)
    finally:
        plan.free()


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-qwen3"])
def test_continuous_batcher_mixes_controlled_and_plain_requests(pkg, orc, make_model, shape):
    m = make_model(shape, pkg.gguf.GGMLType.Q8_0, ctx=64, seed=23)
    V = m.configuration.vocab_size
    eng = pkg.engine
    llama = eng.loop_for(m.model_type) is eng.generate_tokens_llama
    reqs = _requests("LLAMA_3" if llama else "QWEN_3", V, seed=9)
    S = lambda **kw: _controls(pkg, **kw)  # noqa: E731
    menu = [(S(top_k=6, repetition_penalty=1.3), 0.9, 0.0), (None, 0.8, 0.9), (S(presence_penalty=1.0, min_p=0.1), 0.0, 0.0), (None, 0.0, 0.0)]

    def make(i):
        c, t, tp = menu[i % 4]
        return pkg.sampler.Sampler(V, t, tp, 500 + i, controls=c, history=reqs[i][2] if c is not None else None)

    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.set_decode_slots(4)
        got = eng.generate_tokens_continuous(plan, m.model_type, reqs, ARRIVALS, [], 30, 64, samplers=[make(i) for i in range(len(reqs))])
        for i, (latest, start, prompt) in enumerate(reqs):
            c, t, tp = menu[i % 4]
            host = _Host(pkg, orc, V, c, t, tp, 500 + i, prompt if c is not None else ())
            kv_rows = len(prompt) if llama else max(len(prompt) - 1, 0)
            seen = [0]

            def forward(tok, pos):
                seen[0] += 1
                lg, am = plan.forward_decode(tok, pos)
                return am if seen[0] <= kv_rows else host.choose(lg)

            plan.kv_reset()
            assert got[i] == eng.loop_for(m.model_type)(forward, latest, start, prompt, [], 30, 64), f"request {i}"
        # two controlled requests alone: each slot's device counts end as its prompt (the history) plus its generated ids
        cb = eng.ContinuousBatcher(plan, m.model_type, [], 30, 64)
        rids = {cb.submit(*reqs[i], sampler=make(i)): i for i in (0, 2)}
        while cb.pending() or cb.running():
            cb.step()
        for slot, (rid, i) in enumerate(rids.items()):
            want = np.bincount(np.array(reqs[i][2] + cb.results[rid], np.int64), minlength=V)
            assert np.array_equal(plan.sample_counts(slot), want), f"request {i}"
    finally:
        plan.free()


@pytest.mark.parametrize("kind", ["fp16", "qwen2moe", "resident"])
def test_other_plan_types_run_slot_minus_one(pkg, orc, make_model, kind):
    if kind == "fp16":
        m = make_model("tiny-llama", pkg.gguf.GGMLType.F16, ctx=64, seed=24)
        plan = pkg.B200MasterPlan.initialize_plan(m)
    elif kind == "qwen2moe":
        m = make_model("tiny-qwen2moe", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=24)
        plan = pkg.B200MasterPlan.initialize_plan(m)
    else:
        m = _kquant_model(pkg, "tiny-llama", ctx=24)
        plan = _resident_plan(pkg, m)
    V = m.configuration.vocab_size
    c = _controls(pkg, top_k=5, repetition_penalty=1.2, frequency_penalty=0.1, logit_bias={4: 1.0})
    try:
        for temp, topp in ((0.0, 0.0), (0.9, 0.9)):
            smp = pkg.sampler.Sampler(V, temp, topp, 9, controls=c, history=[4, 4])
            plan.kv_reset()
            toks = [2]
            for p in range(8):
                toks.append(smp.sample_token(plan, toks[-1], p))
            counts = plan.sample_counts(-1)
            host = _Host(pkg, orc, V, c, temp, topp, 9, [4, 4])
            assert toks[1:] == _host_chain(plan, host, 2, 8), (kind, temp)
            assert np.array_equal(counts, host.counts), kind
    finally:
        plan.free()


def test_logprobs_and_logits_stay_raw(pkg, orc, make_model):
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=25)
    V = m.configuration.vocab_size
    c = _controls(pkg, top_k=3, repetition_penalty=2.0, logit_bias={0: 1.0})
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        runs = []
        for on in (False, True):
            plan.set_logprobs(5 if on else -1)
            smp = pkg.sampler.Sampler(V, 0.8, 0.0, 4, controls=c)
            plan.kv_reset()
            toks, rows = [1], []
            for p in range(K):
                toks.append(smp.sample_token(plan, toks[-1], p))
                if on:
                    rows.append(plan.last_logprobs())
            runs.append((toks, rows))
        assert runs[0][0] == runs[1][0]
        plan.set_prefill_mode("exact")
        plan.kv_reset()
        lp, _ = plan.score_tokens(runs[1][0][:K], 0, np.array(runs[1][0][1:], np.int32))
        chosen = np.concatenate([r[0] for r in runs[1][1]])
        assert np.array_equal(chosen.view(np.uint64), lp.view(np.uint64)), "chosen is the raw model's log-probability"
        # batched rows: the logits output is the raw row and the logprobs the raw values
        plan.set_decode_slots(2)
        plan.set_sampling_controls(0, c)
        plan.slot_reset(0)
        plan.slot_reset(1)
        ids, lg = plan.forward_decode_batch([0, 1], [1, 1], [0, 0], [(0.0, 0.0, 0.0), (0.0, 0.0, 0.0)], logits=True)
        plan.kv_reset()
        raw, _ = plan.forward_decode(1, 0)
        assert np.array_equal(lg[0].view(np.uint32), raw.view(np.uint32)) and np.array_equal(lg[1].view(np.uint32), raw.view(np.uint32))
        want0 = orc.argmax(sco.modify(raw, np.zeros(V, int), 3, 0.0, 2.0, 0.0, 0.0, {0: 1.0}))
        assert list(ids) == [want0, orc.argmax(raw)]
    finally:
        plan.free()


def test_refusals_name_their_reason_and_leave_the_plan_decoding(pkg, make_model):
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=26)
    V = m.configuration.vocab_size
    S = lambda **kw: _controls(pkg, **kw)  # noqa: E731
    N = pkg.native
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.kv_reset()
        ref = [plan.forward_decode(t, p)[1] for p, t in enumerate([1, 2, 3])]
        with pytest.raises(N.B200Error, match="STATE.*set_sampling_controls"):
            plan.set_sample_history(-1, [1])
        with pytest.raises(N.B200Error, match="STATE"):
            plan.sample_counts(-1)
        bad = {"top_k": S(top_k=V + 1), "min_p": S(min_p=2.0), "repetition_penalty": S(repetition_penalty=0.0),
               "frequency_penalty": S(frequency_penalty=float("nan")), "presence_penalty": S(presence_penalty=float("inf")),
               "out of range": S(logit_bias={V: 1.0}), "not finite": S(logit_bias={1: float("nan")})}
        for why, c in bad.items():
            with pytest.raises(N.B200Error, match=f"BAD_ARG.*{why}"):
                plan.set_sampling_controls(-1, c)
        with pytest.raises(N.B200Error, match="BAD_ARG.*slot 0 out of range"):
            plan.set_sampling_controls(0, S())
        plan.set_sampling_controls(-1, S(top_k=2))
        with pytest.raises(N.B200Error, match="BAD_ARG.*history token 1"):
            plan.set_sample_history(-1, [1, V])
        plan.set_decode_slots(2)
        plan.set_sampling_controls(1, S(top_k=2))
        for s in (0, 1):
            plan.slot_reset(s)
        with pytest.raises(N.B200Error, match="BAD_ARG.*row 1: slot 1 has sampling controls"):
            plan.forward_step([(1, 1, 0, 1), (1, 2, 1, 1)])
        plan.forward_step([(0, 1, 0, 1), (0, 2, 1, 1)])  # a slot without controls may emit twice
        plan.set_sampling_controls(-1, None)
        plan.set_decode_slots(0)
        plan.kv_reset()
        assert [plan.forward_decode(t, p)[1] for p, t in enumerate([1, 2, 3])] == ref
        assert plan.forward_decode_sample(1, 0, 0.0, 0.0, 0.0) == ref[0]
    finally:
        plan.free()


def test_plain_sampler_after_a_controlled_one_samples_the_raw_model(pkg, orc, make_model):
    """One plan, slot -1: a controlled sampler, then a plain sampled one, then the controlled one again after kv_reset.  The plain
    run equals the plain host loop; the controlled runs equal the host loop with the sampler's history plus its earlier ids."""
    m = make_model("tiny-llama", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=27)
    V = m.configuration.vocab_size
    c = _controls(pkg, top_k=3, repetition_penalty=1.8, presence_penalty=0.5, logit_bias={4: 1.0})
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        ctl = pkg.sampler.Sampler(V, 0.9, 0.0, 11, controls=c, history=[4])
        host_ctl = _Host(pkg, orc, V, c, 0.9, 0.0, 11, [4])

        def run(smp, first=1):
            plan.kv_reset()
            toks = [first]
            for p in range(K):
                toks.append(smp.sample_token(plan, toks[-1], p))
            return toks[1:]

        assert run(ctl) == _host_chain(plan, host_ctl, 1)
        for temp, topp in ((0.9, 0.0), (1.0, 0.9), (0.0, 0.0)):
            plain = pkg.sampler.Sampler(V, temp, topp, 12)
            assert run(plain, 2) == _host_chain(plan, _Host(pkg, orc, V, None, temp, topp, 12), 2), (temp, topp)
            assert plan.sampling_controls(-1) is None
        got = run(ctl, 3)
        assert got == _host_chain(plan, host_ctl, 3)  # host_ctl's counts carry its first run, as the sampler's do
        assert np.array_equal(np.bincount([4] + ctl.counted[1:], minlength=V), host_ctl.counts)
    finally:
        plan.free()


def test_tensor_parallel_plan_refuses_controls(pkg, make_model):
    """Rank 0 of a two-way tensor-parallel plan, created without its peer: every sampling-control call names the single-GPU rule."""
    m = make_model("tiny-qwen3", pkg.gguf.GGMLType.Q8_0, ctx=64, seed=28)
    cfg = pkg.plan.make_config(m)
    cfg.tp_rank, cfg.tp_size = 0, 2
    plan = pkg.native.NativePlan(cfg, m.tensors, 0, 0)
    try:
        for call in (lambda: plan.set_sampling_controls(-1, _controls(pkg, top_k=2)), lambda: plan.set_sampling_controls(-1, None),
                     lambda: plan.set_sample_history(-1, [1]), lambda: plan.sample_counts(-1)):
            with pytest.raises(pkg.native.UnsupportedOperation, match="single-GPU"):
                call()
    finally:
        plan.free()
