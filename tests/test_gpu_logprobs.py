"""GPU tests of generated-token log-probabilities (b200_set_logprobs, csrc/logprobs.cuh) on every call that emits ids.
Bar: chosen bit-equal to b200_score_tokens (exact mode) of the same sequence, top ids equal to the numpy restatement over the
call's own logits (test_logprobs_host.logprob_rows), top log-probabilities within 1e-9 of it and bit-equal across calls and decode
modes, top_ids[:, 0] the greedy id, and every id the same with logprobs on and off.  The refusal on tensor-parallel plans is covered
by review only: such a plan needs its peers attached before any call."""
import numpy as np
import pytest

import hostile
from test_logprobs_host import logprob_rows

pytestmark = pytest.mark.gpu

G = hostile.G
N = 5
K = 10  # positions per sequence


def _bits(a):
    return np.asarray(a, np.float64).view(np.uint64)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _decode_modes(pkg, plan):
    out = []
    for mode in ("graph", "persistent"):
        try:
            plan.set_decode_mode(mode)
            out.append(mode)
        except pkg.native.B200Error:
            pass
    return out


def _greedy_chain(plan, start_tok=1):
    """forward_decode from position 0: (inputs, ids, logits, chosen, top ids, top logprobs)."""
    plan.kv_reset()
    toks, ids, lgs, rows = [start_tok], [], [], []
    for p in range(K):
        lg, am = plan.forward_decode(toks[-1], p)
        rows.append(plan.last_logprobs())
        ids.append(am)
        lgs.append(lg)
        toks.append(am)
    c = np.concatenate([r[0] for r in rows])
    ti = np.concatenate([r[1] for r in rows])
    tl = np.concatenate([r[2] for r in rows])
    return np.array(toks[:K], np.int32), np.array(ids, np.int32), np.stack(lgs), c, ti, tl


def _check_restatement(lgs, ids, c, ti, tl):
    rc, ri, rl = logprob_rows(lgs, ids, ti.shape[1])
    assert np.array_equal(ti, ri), f"top ids differ: {ti[:2]} vs {ri[:2]}"
    assert np.nanmax(np.abs(tl - rl)) <= 1e-9 and np.nanmax(np.abs(c - rc)) <= 1e-9


def _score(plan, inputs, targets):
    plan.set_prefill_mode("exact")
    plan.kv_reset()
    lp, _ = plan.score_tokens(inputs, 0, targets)
    return lp


SHAPES = [("tiny-llama", G.Q8_0), ("tiny-qwen3", G.Q8_0), ("tiny-qwen2", G.Q8_0), ("tiny-phi3", G.Q8_0), ("tiny-granite", G.Q8_0),
          ("tiny-devstral", G.Q8_0), ("tiny-llama-vocab128k", G.Q8_0), ("tiny-qwen3-vocab152k", G.Q8_0), ("tiny-llama-vocab509", G.Q8_0),
          ("tiny-qwen2moe", G.Q8_0), ("tiny-llama", G.F16)]


@pytest.mark.parametrize("shape,quant", SHAPES)
def test_every_emitting_call(pkg, make_model, shape, quant):
    m = make_model(shape, quant, ctx=64, seed=5)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=32)
    try:
        plan.set_logprobs(N)
        inputs, ids, lgs, c, ti, tl = _greedy_chain(plan)
        _check_restatement(lgs, ids, c, ti, tl)
        assert np.array_equal(ti[:, 0], ids)
        assert _same(c, _score(plan, inputs, ids)), "chosen differs from score_tokens"
        plan.set_logprobs(N)  # score_tokens leaves the table alone; this empties it
        for mode in _decode_modes(pkg, plan):
            plan.set_decode_mode(mode)
            _, ids2, _, c2, ti2, tl2 = _greedy_chain(plan)
            assert np.array_equal(ids2, ids) and _same(c2, c) and np.array_equal(ti2, ti) and _same(tl2, tl), mode
            plan.kv_reset()
            seq, _ = plan.decode_sequence(inputs[:1], K, 0, feedback=True)
            sc, si, sl = plan.last_logprobs()
            assert np.array_equal(seq, ids) and _same(sc, c) and np.array_equal(si, ti) and _same(sl, tl), mode
            # sampled rows: the same ids with logprobs on and off, and chosen is the sampled id's value
            u = np.random.default_rng(1).random(K).astype(np.float32)
            runs = []
            for on in (False, True):
                plan.set_logprobs(N if on else -1)
                plan.kv_reset()
                out, rows = [], []
                for p in range(K):
                    out.append(plan.forward_decode_sample(int(inputs[p]), p, 0.9, 0.9 if p % 2 else 0.0, float(u[p])))
                    if on:
                        rows.append(plan.last_logprobs())
                runs.append((out, rows))
            assert runs[0][0] == runs[1][0], mode
            sampled_c = np.concatenate([r[0] for r in runs[1][1]])
            assert _same(sampled_c, _score(plan, inputs, np.array(runs[1][0], np.int32))), mode
            assert np.array_equal(np.concatenate([r[1] for r in runs[1][1]]), ti), mode  # the same rows: the inputs are fixed
        if plan.decode_multi_rows() > 0:
            _check_batched(plan, inputs, ids, c, ti, tl)
    finally:
        plan.free()


def _check_batched(plan, inputs, ids, c, ti, tl):
    plan.set_decode_slots(3)
    plan.set_logprobs(N)
    # two slots run the same sequence, greedy; rows in call order
    for s in (0, 1):
        plan.slot_reset(s)
    for p in range(K):
        b_ids, lg = plan.forward_decode_batch([1, 0], [inputs[p]] * 2, [p, p], logits=True)
        bc, bi, bl = plan.last_logprobs()
        assert list(b_ids) == [ids[p]] * 2 and _same(bc, [c[p]] * 2) and np.array_equal(bi, ti[[p, p]]) and _same(bl, tl[[p, p]])
    # a mixed batch with sampled rows: the same ids on and off, chosen the sampled id's value
    u = np.random.default_rng(2).random((K, 3)).astype(np.float32)
    runs = []
    for on in (False, True):
        plan.set_logprobs(N if on else -1)
        for s in (0, 1, 2):
            plan.slot_reset(s)
        out, rows = [], []
        for p in range(K):
            smp = [(0.0, 0.0, 0.0), (0.8, 0.0, u[p, 1]), (1.1, 0.85, u[p, 2])]
            b_ids, _ = plan.forward_decode_batch([0, 1, 2], [inputs[p]] * 3, [p] * 3, smp)
            out.append(list(b_ids))
            if on:
                rows.append(plan.last_logprobs())
        runs.append((out, rows))
    assert runs[0][0] == runs[1][0]
    for j in range(3):
        got = np.array([r[0][j] for r in runs[1][1]])
        want = c if j == 0 else _score(plan, inputs, np.array([o[j] for o in runs[1][0]], np.int32))
        assert _same(got, want), f"row {j}"
        assert np.array_equal(np.stack([r[1][j] for r in runs[1][1]]), ti)
    plan.set_logprobs(N)
    # forward_decode_multi on the plan's own cache
    plan.kv_reset()
    m_ids, _ = plan.forward_decode_multi(-1, inputs[:4], 0)
    mc, mi, ml = plan.last_logprobs()
    assert list(m_ids) == list(ids[:4]) and _same(mc, c[:4]) and np.array_equal(mi, ti[:4]) and _same(ml, tl[:4])
    # forward_step: a K/V-only row reports NaN and -1
    plan.slot_reset(2)
    s_ids, _ = plan.forward_step([(2, int(inputs[0]), 0, 0), (2, int(inputs[1]), 1, 1)])
    fc, fi, fl = plan.last_logprobs()
    assert s_ids[0] == -1 and np.isnan(fc[0]) and (fi[0] == -1).all() and np.isnan(fl[0]).all()
    assert s_ids[1] == ids[1] and _same(fc[1:], c[1:2]) and np.array_equal(fi[1], ti[1]) and _same(fl[1], tl[1])
    plan.set_decode_slots(0)


@pytest.mark.parametrize("shape", ["tiny-llama", "tiny-llama-vocab128k"])
@pytest.mark.parametrize("kind", hostile.TIE_KINDS)
def test_tied_logits_take_the_lower_index(pkg, shape, kind):
    m = hostile.tied_logits(shape, G.Q8_0, kind)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        plan.set_logprobs(20)
        _, ids, lgs, c, ti, tl = _greedy_chain(plan, 4)
        _check_restatement(lgs, ids, c, ti, tl)
        assert np.array_equal(ti[:, 0], ids)
    finally:
        plan.free()


def test_values_of_n_and_refusals(pkg, make_model):
    m = make_model("tiny-llama", G.Q8_0, ctx=64, seed=5)
    plan = pkg.B200MasterPlan.initialize_plan(m)
    try:
        for bad in (21, -2):
            with pytest.raises(pkg.native.B200Error, match="BAD_ARG"):
                plan.set_logprobs(bad)
        with pytest.raises(pkg.native.B200Error, match="STATE"):
            plan.last_logprobs()
        ref = None
        for n in (0, 1, 20):
            plan.set_logprobs(n)
            plan.kv_reset()
            _, am = plan.forward_decode(1, 0)
            c, ti, tl = plan.last_logprobs()
            assert c.shape == (1,) and ti.shape == (1, n) and tl.shape == (1, n)
            if n:
                assert ti[0, 0] == am
            assert ref is None or _same(c, ref)
            ref = c
    finally:
        plan.free()


def test_switched_off_is_never_switched_on(pkg, make_model):
    """After set_logprobs(-1): ids, logits and launch counts bit-equal to a plan that never had logprobs on."""
    m = make_model("tiny-llama", G.Q8_0, ctx=64, seed=5)
    plans = [pkg.B200MasterPlan.initialize_plan(m) for _ in range(2)]
    try:
        plans[1].set_logprobs(20)
        plans[1].forward_decode(1, 0)
        plans[1].set_logprobs(-1)
        res = []
        for plan in plans:
            plan.kv_reset()
            r = [plan.forward_decode(1, 0), plan.decode_sequence([3], 6, 1, feedback=True)[0], plan.decode_info()]
            plan.set_decode_slots(2)
            plan.slot_reset(0)
            r += [plan.forward_decode_batch([0], [5], [0], [(0.7, 0.9, 0.3)], logits=True), plan.batch_info()[:2]]
            res.append(r)
        a, b = res
        assert np.array_equal(a[0][0].view(np.uint32), b[0][0].view(np.uint32)) and a[0][1] == b[0][1]
        assert np.array_equal(a[1], b[1]) and a[2] == b[2] and a[4] == b[4]
        assert np.array_equal(a[3][0], b[3][0]) and np.array_equal(a[3][1].view(np.uint32), b[3][1].view(np.uint32))
    finally:
        for plan in plans:
            plan.free()


def test_engine_entries_are_the_scores(pkg, make_model):
    """The engine loops' entries against engine.score_sequence over latest + prompt + generated, at the generated positions."""
    eng = pkg.engine
    m = make_model("tiny-llama", G.Q8_0, ctx=64, seed=5)
    plan = pkg.B200MasterPlan.initialize_plan(m, prefill_batch_size=16)
    stop, budget = [10 ** 6], 24
    reqs = [(1, 0, [5, 6, 7]), (2, 0, [9, 9, 3, 4, 8])]
    try:
        plan.set_decode_slots(2)

        def check(latest, prompt, gen, entries):
            seq = [latest] + list(prompt) + list(gen)
            plan.set_prefill_mode("exact")
            plan.kv_reset()
            lp, _ = eng.score_sequence(plan, seq, 0)
            first = len(prompt)  # the first generated id is the target of row len(prompt)
            assert len(entries) == len(gen)
            assert _same([e[0] for e in entries], lp[first:first + len(gen)])
            assert [e[1][0][0] for e in entries] == list(gen)  # greedy: the top alternative is the id

        runs = {}
        for on in (False, True):
            plan.set_logprobs(N if on else -1)
            lp = [] if on else None
            out = {"batch": (eng.generate_tokens_batch(plan, "LLAMA_3", reqs, stop, budget, 64, logprobs=lp), lp)}
            lp = [] if on else None
            out["batch_prefill"] = (eng.generate_tokens_batch_prefill(plan, "LLAMA_3", reqs, stop, budget, 64, 4, logprobs=lp), lp)
            lp = [] if on else None
            out["continuous"] = (eng.generate_tokens_continuous(plan, "LLAMA_3", reqs, [0, 1], stop, budget, 64, logprobs=lp), lp)
            lp = [] if on else None
            plan.kv_reset()
            out["llama_batch_prefill"] = ([eng.generate_tokens_llama_batch_prefill(plan, 1, 0, [5, 6, 7], stop, budget, 64, 4, logprobs=lp)], [lp])
            lp = [] if on else None
            plan.kv_reset()
            out["lookahead"] = ([eng.generate_tokens_lookahead(plan, "LLAMA_3", 1, 0, [5, 6, 7], stop, budget, 64, logprobs=lp)], [lp])
            runs[on] = out
        for name, (ids, lps) in runs[True].items():
            assert ids == runs[False][name][0], name
            for i, gen in enumerate(ids):
                latest, _, prompt = reqs[i] if len(ids) > 1 else reqs[0]
                check(latest, prompt, gen, lps[i])
    finally:
        plan.free()


SCORE_THREADS, LOGPROB_CAND = 256, 1024  # csrc/score.cuh, csrc/logprobs.cuh


def _keys(row):
    """logprob_key of every entry (csrc/logprobs.cuh) as Python ints."""
    b = np.where(row == 0, np.float32(0), row).view(np.uint32).astype(np.uint64)
    hi = np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000)
    hi = np.where(row > -np.inf, hi, 0)
    return (hi << np.uint64(32)) | (~np.arange(len(row), dtype=np.uint64) & 0xFFFFFFFF)


def _candidates(row, n_top):
    """How many keys k_token_logprobs puts on its candidate list: those >= the n_top-th largest of the per-thread maxima."""
    k = _keys(row)
    mx = np.array([k[t::SCORE_THREADS].max() if t < len(k) else 0 for t in range(SCORE_THREADS)], np.uint64)
    T = np.sort(mx)[::-1][n_top - 1]
    return int((k >= T).sum())


def _close(got, want):
    """NaN where want is NaN, infinities equal, everything else within 1e-9."""
    nan = np.isnan(want)
    if not np.array_equal(np.isnan(got), nan):
        return False
    g, w = got[~nan], want[~nan]
    inf = np.isinf(w)
    return np.array_equal(g[inf], w[inf]) and bool((np.abs(g[~inf] - w[~inf]) <= 1e-9).all())


@pytest.mark.parametrize("V", [509, 128256])
def test_kernel_on_hostile_rows(pkg, V):
    """k_token_logprobs alone: the candidate list, its overflow fallback, ties of equal values and of -0 / +0, rows without a finite
    maximum.  The fallback needs more than LOGPROB_CAND keys at or above the threshold, and only the n_top slices (of ceil(V / 256)
    entries each) whose maximum reaches it contribute: at V = 128256 three slices lying wholly above every other entry do."""
    rng = np.random.default_rng(V)
    rows = {"random": (rng.standard_normal(V) * 3).astype(np.float32)}
    r = (rng.standard_normal(V) - 20).astype(np.float32)
    r[::256] = rng.standard_normal(len(r[::256])).astype(np.float32)  # one slice of the 256-thread layout owns the top
    rows["one_slice"] = r
    r = (rng.standard_normal(V) - 20).astype(np.float32)
    for t in range(3):
        r[t::256] = rng.standard_normal(len(r[t::256])).astype(np.float32)
    rows["three_slices"] = r
    overflow = _candidates(r, 20) > LOGPROB_CAND
    assert overflow == (V == 128256), _candidates(r, 20)
    rows["ties"] = np.round(rng.standard_normal(V)).astype(np.float32)
    z = np.zeros(V, np.float32)
    z[1::2] = -0.0
    rows["signed_zero"] = z
    rows["all_minus_inf"] = np.full(V, -np.inf, np.float32)
    r = np.full(V, -np.inf, np.float32)
    r[[7, V - 1, 3]] = [1.0, 1.0, np.nan]
    rows["few_finite"] = r
    for name, row in rows.items():
        for n_top in (1, 20):
            c, ids, lps, _ = pkg.native.test_logprobs(row, 3, n_top)
            rc, ri, rl = logprob_rows(row[None], np.array([3]), n_top)
            assert np.array_equal(ids, ri[0]), (name, n_top)
            assert _close(np.append(lps, c), np.append(rl[0], rc[0])), (name, n_top)  # the top values and chosen
