"""Host checks of the sampling controls: the numpy restatement (sampling_controls_oracle) against an independent formulation -- a
full sort for top-k, a per-element Python loop for the bias and penalties -- on random and adversarial rows, and
sampler.SamplingControls' validation against the C call's rules."""
import math

import numpy as np
import pytest

import sampling_controls_oracle as sco

F = np.float32


def _independent(logits, counts, top_k, min_p, rep, freq, pres, bias):
    lg = [F(x) for x in logits]
    for i, b in (bias or {}).items():
        lg[i] = F(lg[i] + F(b))
    for i, c in enumerate(counts):
        if c > 0:
            x = lg[i]
            x = F(x * F(rep)) if x <= 0 else F(x / F(rep))
            lg[i] = F(x - F(F(F(c) * F(freq)) + F(pres)))
    m = max(lg)
    order = sorted(lg, reverse=True)
    vk = order[top_k - 1] if 0 < top_k < len(lg) else -math.inf
    thr = F(m + F(math.log(min_p))) if min_p > 0 else -math.inf
    return np.array([x if (x >= vk and x >= thr) else -np.inf for x in lg], dtype=F)


def _rows(V, rng):
    r = {"random": (rng.standard_normal(V) * 4).astype(F)}
    r["ties"] = np.round(rng.standard_normal(V) * 2).astype(F)  # many ties around every v_k
    r["negative"] = -np.abs(rng.standard_normal(V)).astype(F)
    z = np.zeros(V, F)
    z[1::2] = -0.0
    r["signed_zero"] = z
    r["flat"] = np.full(V, 1.5, F)
    return r


CASES = [dict(top_k=0, min_p=0.0, rep=1.0, freq=0.0, pres=0.0, bias=None),
         dict(top_k=1, min_p=0.0, rep=1.0, freq=0.0, pres=0.0, bias=None),
         dict(top_k=7, min_p=0.0, rep=1.0, freq=0.0, pres=0.0, bias=None),
         dict(top_k=10 ** 6, min_p=0.0, rep=1.0, freq=0.0, pres=0.0, bias=None),  # top_k >= vocab: off
         dict(top_k=0, min_p=1.0, rep=1.0, freq=0.0, pres=0.0, bias=None),
         dict(top_k=0, min_p=0.05, rep=1.3, freq=0.0, pres=0.0, bias=None),
         dict(top_k=0, min_p=0.0, rep=0.7, freq=0.11, pres=0.4, bias=None),
         dict(top_k=5, min_p=0.2, rep=1.1, freq=-0.3, pres=0.25, bias="argmax")]


@pytest.mark.parametrize("V", [1, 2, 512, 4099])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_restatement_matches_independent_formulation(V, case):
    rng = np.random.default_rng(V * 31 + case)
    k = dict(CASES[case])
    for name, row in _rows(V, rng).items():
        counts = rng.integers(0, 3, V) * (rng.random(V) < 0.3)
        counts[: min(3, V)] = [4000, 0, 2][: min(3, V)]
        bias = None
        if k["bias"] == "argmax":
            bias = {int(np.argmax(row)): -100.0, int(rng.integers(V)): 2.5} if V > 1 else {0: -100.0}
        got = sco.modify(row, counts, k["top_k"], k["min_p"], k["rep"], k["freq"], k["pres"], bias)
        want = _independent(row, counts, k["top_k"], k["min_p"], k["rep"], k["freq"], k["pres"], bias)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, k)
        assert np.isfinite(got).any(), name  # the maximum always survives


def test_ties_at_v_k_are_all_kept():
    row = np.array([3, 1, 2, 2, 2, 0], F)
    got = sco.modify(row, np.zeros(6, int), top_k=2)
    assert list(np.isfinite(got)) == [True, False, True, True, True, False]


def test_neutral_controls_leave_the_row():
    row = (np.random.default_rng(0).standard_normal(1000) * 3).astype(F)
    got = sco.modify(row, np.random.default_rng(1).integers(0, 5, 1000))
    assert np.array_equal(got.view(np.uint32), row.view(np.uint32))


def test_controls_validate_like_the_c_call(pkg):
    S = pkg.sampler.SamplingControls
    ok = [S(), S(top_k=10), S(min_p=1.0), S(repetition_penalty=0.5, frequency_penalty=-2, presence_penalty=2), S(logit_bias={0: -100.0, 9: 1.0})]
    for c in ok:
        assert c.validate(10) is c
    bad = [S(top_k=-1), S(top_k=11), S(min_p=-0.1), S(min_p=1.5), S(min_p=math.nan), S(repetition_penalty=0.0),
           S(repetition_penalty=math.inf), S(frequency_penalty=math.nan), S(presence_penalty=-math.inf), S(logit_bias={10: 1.0}),
           S(logit_bias={-1: 1.0}), S(logit_bias={3: math.inf}), S(logit_bias={i: 1.0 for i in range(1025)})]
    for c in bad:
        with pytest.raises(ValueError):
            c.validate(10 if not c.logit_bias or len(c.logit_bias) < 1000 else 5000)
    with pytest.raises(ValueError):
        pkg.sampler.Sampler(10, 0.0, 0.0, 1, controls=S(top_k=11))
    with pytest.raises(ValueError):
        pkg.sampler.Sampler(10, 0.0, 0.0, 1, controls=S(), history=[10])


class _FakeNative:
    """Stands in for native.NativePlan under a real B200MasterPlan: records the calls, emits 7 from the device sampler and 3 as argmax."""

    def __init__(self):
        self.calls = []

    def set_sampling_controls(self, slot, c):
        self.calls.append(("controls", slot, c))

    def set_sample_history(self, slot, t):
        self.calls.append(("history", slot, list(t)))

    def forward_decode_sample(self, token, position, temperature, topp, u, want_info=False):
        self.calls.append(("sample", token, position, temperature, topp, u))
        return 7

    def forward_decode(self, token, position, want_logits=True, want_argmax=True):
        self.calls.append(("decode", token, position))
        return None, 3

    def kv_reset(self):
        self.calls.append(("kv_reset",))


def _plan(pkg):
    plan = object.__new__(pkg.B200MasterPlan)  # its slot bookkeeping over a recording native plan
    plan._native, plan._controls = _FakeNative(), {}
    return plan


def test_sampler_routes_controls_through_the_device_sampler(pkg):
    smp = pkg.sampler
    c = smp.SamplingControls(top_k=4)
    greedy = smp.Sampler(10, 0.0, 0.0, 1, controls=c, history=[1, 1, 2])
    plan = _plan(pkg)
    assert greedy.sample_token(plan, 5, 0) == 7 and greedy.sample_token(plan, 7, 1) == 7
    assert plan._native.calls == [("controls", -1, c), ("history", -1, [1, 1, 2]), ("sample", 5, 0, 0.0, 0.0, 0.0), ("sample", 7, 1, 0.0, 0.0, 0.0)]
    hot = smp.Sampler(10, 0.8, 0.9, 42, controls=c)
    ref = smp.L32X64MixRandom(42)
    plan = _plan(pkg)
    hot.sample_token(plan, 5, 0)
    hot.sample_token(plan, 7, 1)
    assert [x[5] for x in plan._native.calls if x[0] == "sample"] == [ref.next_float1(), ref.next_float1()]
    plain = smp.Sampler(10, 0.0, 0.0, 1)  # no controls on the plan: the plan's argmax, as before
    plan = _plan(pkg)
    assert plain.sample_token(plan, 5, 0) == 3 and plan._native.calls == [("decode", 5, 0)]


def test_slot_minus_one_follows_the_sampler_in_use(pkg):
    """A plain sampler after a controlled one turns the controls off; two controlled samplers take turns with their own controls and
    counts; after kv_reset a controlled sampler installs its controls and counts (history + emitted ids) again."""
    smp = pkg.sampler
    c1, c2 = smp.SamplingControls(top_k=4), smp.SamplingControls(repetition_penalty=1.3)
    a = smp.Sampler(10, 0.0, 0.0, 1, controls=c1, history=[1])
    b = smp.Sampler(10, 0.0, 0.0, 1, controls=c2, history=[2])
    plain = smp.Sampler(10, 0.8, 0.0, 5)
    plan = _plan(pkg)
    calls = plan._native.calls
    a.sample_token(plan, 5, 0)
    del calls[:]
    plain.sample_token(plan, 7, 1)
    plain.sample_token(plan, 7, 2)
    assert [x[:3] for x in calls] == [("controls", -1, None), ("sample", 7, 1), ("sample", 7, 2)]
    assert plan.sampling_controls(-1) is None
    del calls[:]
    a.sample_token(plan, 7, 1)
    b.sample_token(plan, 7, 1)
    a.sample_token(plan, 7, 2)
    a.sample_token(plan, 7, 3)
    assert [x for x in calls if x[0] != "sample"] == [("controls", -1, c1), ("history", -1, [1, 7]), ("controls", -1, c2), ("history", -1, [2]),
                                                       ("controls", -1, c1), ("history", -1, [1, 7, 7])]
    del calls[:]
    plan.kv_reset()
    a.sample_token(plan, 7, 0)
    assert [x for x in calls if x[0] != "sample"] == [("kv_reset",), ("controls", -1, c1), ("history", -1, [1, 7, 7, 7, 7])]
    del calls[:]
    plan.set_sampling_controls(-1, c2)  # the caller's own controls: a plain sampler turns them off too
    plain.sample_token(plan, 7, 1)
    assert calls[1] == ("controls", -1, None)


def test_abi_is_exported_and_wrapped(pkg):
    import inspect
    n = pkg.native
    names = {"b200_set_sampling_controls", "b200_set_sample_history", "b200_read_sample_counts", "b200_test_sample_controls"}
    assert names <= set(n.EXPORTS)
    for cls in (n.NativePlan, pkg.B200MasterPlan):
        assert list(inspect.signature(cls.set_sampling_controls).parameters)[:3] == ["self", "slot", "controls"]
        assert list(inspect.signature(cls.set_sample_history).parameters) == ["self", "slot", "tokens"]
        assert list(inspect.signature(cls.sample_counts).parameters) == ["self", "slot"]
    assert [f[0] for f in n.SamplingControlsC._fields_] == ["top_k", "min_p", "repetition_penalty", "frequency_penalty", "presence_penalty",
                                                            "n_bias", "bias_ids", "bias_values"]
