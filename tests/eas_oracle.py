"""Float64 reference for the EAS-Emb key gradient: the oracle's teacher-forced decode loop with the logit key replaced.

`O.teacher_forced_logprobs` reads the logit key from `O.precompute_cache`; `teacher_forced_logprobs_with_key` runs it
with that one entry of the cache replaced by a given per-instance key L [B, N, E] (batchified like the encoder output
for multistart rows).  A float64 leaf L then gives d(loss)/dL by autograd through the reference-restated decoder
(rl4co/models/zoo/eas/search.py:172-177 makes exactly this tensor the parameter)."""

from oracle import am_rollout_oracle as O


def teacher_forced_logprobs_with_key(weights, env_name, inst, h, acts, logit_key, num_starts=1, **kw):
    key = O.batchify(logit_key, num_starts) if num_starts > 1 else logit_key
    original = O.precompute_cache

    def with_key(*a, **k):
        cache = dict(original(*a, **k))
        cache["logit_key"] = key
        return cache

    O.precompute_cache = with_key
    try:
        return O.teacher_forced_logprobs(weights, env_name, inst, h, acts, num_starts=num_starts, **kw)
    finally:
        O.precompute_cache = original
