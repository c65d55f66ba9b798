"""Rollout-side glue restated in NumPy: running mean / std, observation normalisation and the categorical policy's
sample / log-prob / entropy.  TEST INFRASTRUCTURE (see oracle/__init__).

Follows
  * ``RunningMeanStd.update / update_from_moments`` ........ xuance/common/statistic_tools.py:117-185
  * ``Agent._process_observation`` .......................... xuance/torch/agents/base/agent.py:262-279 (EPS = 1e-8,
    xuance/common/common_tools.py:8)
  * ``CategoricalDistribution`` ............................. xuance/torch/rl_models/modules/distributions.py:128-162
    (torch.distributions.Categorical: logits - logsumexp, probs = softmax, entropy = -sum p log p, argmax of probs)
The draw itself: the reference calls ``Categorical.sample()`` (torch.multinomial on torch's RNG), whose stream cannot be
shared with a CUDA kernel; as for PER the parity definition is on SUPPLIED uniforms - the inverse CDF in action-index
order, which samples the same distribution.
"""
import numpy as np

EPS = 1e-8


class RunningMeanStdOracle:
    """statistic_tools.py:83-185 for a non-dict shape, no MPI.  float32 arrays, Python-float count (a weak scalar under
    NumPy >= 2, so every product below is evaluated in float32 exactly as in the reference)."""

    def __init__(self, shape, epsilon=1e-4):
        self.mean = np.zeros(shape, np.float32)
        self.var = np.ones(shape, np.float32)
        self.count = epsilon

    @property
    def std(self):
        return np.sqrt(self.var)

    def update(self, x):  # :117-145
        batch_mean, batch_std, batch_count = np.mean(x, axis=0), np.std(x, axis=0), x.shape[0]
        self.update_from_moments(batch_mean, np.square(batch_std), batch_count)

    def update_from_moments(self, batch_mean, batch_var, batch_count):  # :147-185
        delta = batch_mean - self.mean
        tot_count = self.count + batch_count
        new_mean = self.mean + delta * batch_count / tot_count
        m_a = self.var * self.count
        m_b = batch_var * batch_count
        m2 = m_a + m_b + np.square(delta) * self.count * batch_count / tot_count
        self.mean, self.var, self.count = new_mean, m2 / tot_count, tot_count


def process_observation(obs, rms, obsnorm_range=5):
    """agent.py:273-276."""
    return np.clip((obs - rms.mean) / (rms.std + EPS), -obsnorm_range, obsnorm_range)


def categorical_terms(logits):
    """float32 log-probabilities, probabilities and entropy of Categorical(logits=...) (distributions.py:136-150)."""
    z = np.asarray(logits, np.float32)
    m = z.max(axis=-1, keepdims=True)
    lse = m + np.log(np.exp(z - m).sum(axis=-1, keepdims=True, dtype=np.float32))
    logp = (z - lse).astype(np.float32)
    p = np.exp(logp)
    return logp, p, -np.where(p > 0, p * logp, np.float32(0)).sum(axis=-1, dtype=np.float32)   # 0 * -inf adds nothing


def categorical_act(logits, uniforms=None, forced_actions=None):
    """Returns (actions int64 [N], logp float32 [N], entropy float32 [N], cdf float32 [N, A]).
    forced_actions: log_prob of given actions (:146-147); uniforms: inverse-CDF draw; neither: argmax of probs (:155-156)."""
    logp, p, ent = categorical_terms(logits)
    N, A = p.shape
    cdf = np.zeros_like(p)
    run = np.zeros(N, np.float32)
    for i in range(A):                      # sequential float32 accumulation in index order
        run = (run + p[:, i]).astype(np.float32)
        cdf[:, i] = run
    if forced_actions is not None:
        a = np.asarray(forced_actions).astype(np.int64)
    elif uniforms is not None:
        u = np.asarray(uniforms, np.float32)[:, None]
        hit = u < cdf
        last_pos = A - 1 - (p > 0)[:, ::-1].argmax(axis=1)     # no prefix passed u: the last category with p > 0
        a = np.where(hit.any(axis=1), hit.argmax(axis=1), last_pos).astype(np.int64)
    else:
        a = p.argmax(axis=1).astype(np.int64)
    return a, logp[np.arange(N), a], ent, cdf
