"""Windowed GAE and n-step return (reference: surreal/learner/ppo.py:355-418, SURVEY Appendix A.1)."""
import torch


def gae_from_values(rewards, values_raw, dones, gamma, lam, horizon=None, norm_adv=True):
    """rewards [B,n] fp32, values_raw [B,n+1] fp32 (critic output BEFORE masking), dones [B,n] fp32.

    ``horizon=None`` (or == n) is the MLP branch (ppo.py:408-418): one advantage / return per
    window.  Otherwise the RNN branch (ppo.py:389-406): ``n-horizon+1`` outputs per window.
    ``gamma``/``lam`` are Python floats exactly as in the learner config.
    """
    B, n = rewards.shape
    idx = torch.tensor(range(n), dtype=rewards.dtype)            # ppo.py:372 (float32 there; float64 inputs: a float64 run)
    g = torch.pow(gamma, idx)                                    # ppo.py:373
    l = torch.pow(lam, idx)                                      # ppo.py:374
    values = values_raw.clone()
    values[:, 1:] *= 1 - dones                                   # ppo.py:387
    tds = rewards + gamma * values[:, 1:] - values[:, :-1]
    if horizon is None or horizon == n:
        returns = torch.sum(g * rewards, 1) + values[:, -1] * (gamma ** n)
        adv = torch.sum(tds * g * l, 1)
        if norm_adv:
            std, mean = adv.std(), adv.mean()
            adv = (adv - mean) / max(std, 1e-4)
        return adv.view(-1, 1), returns.view(-1, 1)
    H = horizon
    E = n - H + 1
    g, l = g[:H], l[:H]
    returns = torch.zeros(B, E, dtype=rewards.dtype)
    advs = torch.zeros(B, E, dtype=rewards.dtype)
    for s in range(E):
        returns[:, s] = torch.sum(g * rewards[:, s:s + H], 1) + values[:, s + H] * (gamma ** H)
        advs[:, s] = torch.sum(tds[:, s:s + H] * g * l, 1)
    if norm_adv:
        std, mean = advs.std(), advs.mean()
        advs = (advs - mean) / max(std, 1e-4)
    return advs, returns


def gae_reference_fp64(rewards, values_raw, dones, gamma, lam, horizon=None, reward_scale=1.0):
    """The same formula evaluated in float64 via the backward recurrence, truncated to ``horizon`` steps.

    ``horizon=None`` (or == n): the MLP branch, adv / ret of shape [B].  Otherwise the RNN branch: [B, E] with
    E = n - horizon + 1, output s being the recurrence over steps s .. s + horizon - 1 bootstrapped from V[s + horizon].
    ``reward_scale`` is applied as the learner applies it (ppo.py:452): the fp32 rewards times the scale, rounded to
    fp32, before anything else.  No advantage normalisation.
    """
    r = rewards.double() if reward_scale == 1.0 else (rewards.float() * reward_scale).double()
    v = values_raw.double().clone()
    v[:, 1:] *= 1 - dones.double()
    B, n = r.shape
    H = n if horizon is None else int(horizon)
    E = n - H + 1
    td = r + gamma * v[:, 1:] - v[:, :-1]
    adv = torch.zeros(B, E, dtype=torch.float64, device=r.device)
    ret = v[:, H:H + E].clone()
    for k in reversed(range(H)):
        adv = td[:, k:k + E] + gamma * lam * adv
        ret = r[:, k:k + E] + gamma * ret
    if horizon is None or H == n:
        return adv[:, 0], ret[:, 0]
    return adv, ret
