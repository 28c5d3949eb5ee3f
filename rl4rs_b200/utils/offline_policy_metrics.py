"""The off-policy estimators of rl4rs/utils/offline_policy_metrics.py, under the reference's names and signatures, on the
host in NumPy / SciPy.  They run once per evaluation epoch on B x T numbers (2048 x 36 at most in the scripts), so there is
no kernel.  Each keeps the reference's arithmetic, quirks included (INTEGRATION.md, "Off-policy evaluation"):

  - where a [0.1, 10] clip is passed (CIPS, SNIPS, DR), the ratios are clipped BEFORE the effective sample size behind the
    t quantile is formed; IPS is unclipped;
  - _calc_sequential_weigths divides the clipped cumulative ratios by B (or their column sums), THEN clips again to >= 0.1;
  - the t quantile has int(n_e) - 1 degrees of freedom (NaN when that is < 1);
  - DR's half-width is scipy.stats.sem of the per-episode estimates;
  - DR and SeqDR are divided by the mean offline return.

Results are (estimate, half-width) pairs; WIPS and SeqDR report a half-width of 0.  Inputs keep their dtypes: the
reference's float32 propensities stay float32 through the ratios, as there.
"""
import numpy as np
import scipy.stats

ALPHA = 0.00125          # the t quantile 1 - ALPHA of the half-widths
CLIP = (0.1, 10)


def _calc_sequential_weigths(policy_prob, behavior_prob, weighted=False, a_min=None, a_max=None):
    """Per-step weights [B, T]: the running product over steps of the (clipped) ratios, divided by B (weighted: by each
    step's column sum), then clipped with the same bounds."""
    ratio = np.asarray(policy_prob) / np.asarray(behavior_prob)
    rho = np.cumprod(np.clip(ratio, a_min, a_max), axis=1)
    ws = rho / (rho.sum(axis=0) if weighted else len(policy_prob))
    return np.clip(ws, a_min, a_max)


def _calc_sample_weigths(policy_prob, behavior_prob, a_min=None, a_max=None):
    """(ratios, effective sample size n_e, t quantile at 1 - ALPHA with int(n_e) - 1 degrees of freedom).  The ratios are
    clipped when a_min is given, before n_e is formed."""
    ratio = np.asarray(policy_prob) / np.asarray(behavior_prob)
    if a_min is not None:
        ratio = np.clip(ratio, a_min, a_max)
    n_e = len(policy_prob) * np.mean(ratio) ** 2 / np.mean(ratio ** 2)
    return ratio, n_e, scipy.stats.t.ppf(1 - ALPHA, df=int(n_e) - 1)


def _half_width(cv, spread, n_e):
    return cv * spread / np.sqrt(int(n_e))


def eval_DM(policy, obs):
    return policy(obs)


def eval_IPS(rewards, policy_prob, behavior_prob):
    """Inverse propensity scoring with unclipped ratios."""
    ratio, n_e, cv = _calc_sample_weigths(policy_prob, behavior_prob)
    weighted = rewards * ratio
    est = np.mean(weighted)
    return est, _half_width(cv, np.sqrt(np.mean((weighted - est) ** 2)), n_e)


def eval_CIPS(rewards, policy_prob, behavior_prob):
    """Capped IPS: the ratios clipped to [0.1, 10]."""
    ratio, n_e, cv = _calc_sample_weigths(policy_prob, behavior_prob, *CLIP)
    weighted = rewards * np.clip(ratio, *CLIP)
    est = np.mean(weighted)
    return est, _half_width(cv, np.sqrt(np.mean((weighted - est) ** 2)), n_e)


def eval_SNIPS(rewards, policy_prob, behavior_prob):
    """Self-normalised IPS over the clipped ratios."""
    ratio, n_e, cv = _calc_sample_weigths(policy_prob, behavior_prob, *CLIP)
    total = np.sum(ratio)
    est = np.sum(rewards * ratio) / total
    var = np.sum((rewards - est) ** 2 * ratio ** 2) / total ** 2
    return est, _half_width(cv, np.sqrt(var), n_e)


def eval_WIPS(step_rewards, policy_prob, behavior_prob, gamma=1.0):
    """Step-wise weighted IS: each step's weight over the mean of the weights up to it, against the logged return."""
    steps = len(step_rewards[0])
    p = _calc_sequential_weigths(policy_prob, behavior_prob, a_min=CLIP[0], a_max=CLIP[1])
    w = np.stack([np.average(p[:, :t + 1], axis=1) for t in range(steps)], axis=1)
    logged, weighted = 0.0, 0.0
    for t in range(steps):
        logged += np.sum(step_rewards[:, t] * gamma ** t)
        weighted += np.sum(p[:, t] / w[:, t] * step_rewards[:, t] * gamma ** t)
    return weighted / np.clip(logged, 1e-8, None), 0


def eval_doubly_robust(action_rhat_rewards, state_rewards, rewards, policy_prob, behavior_prob):
    """Episode-level doubly robust: state_rewards + ratio (rewards - action_rhat_rewards), its mean over the mean logged
    return, and scipy.stats.sem of the per-episode terms."""
    ratio, n_e, cv = _calc_sample_weigths(policy_prob, behavior_prob, *CLIP)
    dr = state_rewards + ratio * (rewards - action_rhat_rewards)
    return np.mean(dr) / np.average(rewards), scipy.stats.sem(dr)


def eval_seq_doubly_robust(action_rhat_rewards, state_rewards, rewards, policy_prob, behavior_prob):
    """Sequential doubly robust, folded from the last step back, over the mean logged return."""
    ws = _calc_sequential_weigths(policy_prob, behavior_prob, a_min=CLIP[0], a_max=CLIP[1])
    steps = len(action_rhat_rewards[0])
    dr = np.zeros(len(action_rhat_rewards))
    for t in range(steps - 1, -1, -1):
        dr = state_rewards[:, t] + ws[:, t] * (rewards[:, t] + dr - action_rhat_rewards[:, t])
    return np.average(dr) / np.mean(np.sum(rewards, axis=1)), 0
