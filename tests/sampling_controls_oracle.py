"""Numpy float32 restatement of the sampling controls (include/b200llama.h, b200_set_sampling_controls): steps 1-4 modify a raw
logits row, step 5 counts the emitted id.  Every operation is one float32 operation, rounded once, as k_sample_ctl evaluates it;
the choice itself is the oracle's (oracle.sample / oracle.argmax) on the modified row."""
import math

import numpy as np

F = np.float32


def min_p_log(min_p: float) -> np.float32:
    """(float)log((double)min_p); -inf for 0."""
    return F(math.log(min_p)) if min_p > 0 else F(-np.inf)


def modify(logits, counts, top_k=0, min_p=0.0, repetition_penalty=1.0, frequency_penalty=0.0, presence_penalty=0.0, logit_bias=None):
    """The modified row (float32, masked entries -inf) of raw logits under the controls and the sequence's counts."""
    lg = np.array(logits, dtype=F, copy=True)
    cnt = np.asarray(counts)
    if logit_bias:  # 1. bias (distinct ids)
        ids = np.fromiter(logit_bias.keys(), dtype=np.int64, count=len(logit_bias))
        lg[ids] = lg[ids] + np.array(list(logit_bias.values()), dtype=F)
    hit = cnt > 0  # 2. penalties
    v = lg[hit]
    v = np.where(v <= 0, v * F(repetition_penalty), v / F(repetition_penalty)).astype(F)
    lg[hit] = v - ((cnt[hit].astype(F) * F(frequency_penalty)) + F(presence_penalty))
    m = lg.max()  # 3. masks, both on the row of step 2
    keep = lg >= F(m + min_p_log(min_p))
    if 0 < top_k < len(lg):
        keep &= lg >= np.partition(lg, len(lg) - top_k)[len(lg) - top_k]
    lg[~keep] = -np.inf
    return lg


def step(orc, logits, counts, controls, temperature, topp, uniform01):
    """Steps 1-5 for one emitting row: (id, modified row); counts (int array) gains the id.  controls: sampler.SamplingControls."""
    row = modify(logits, counts, controls.top_k, controls.min_p, controls.repetition_penalty, controls.frequency_penalty,
                 controls.presence_penalty, controls.logit_bias)
    tok = orc.argmax(row) if temperature == 0.0 else orc.sample(row, temperature, topp, uniform01)
    counts[tok] += 1
    return tok, row
