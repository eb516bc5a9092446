"""TEST INFRASTRUCTURE -- float64 restatement of the reference DQN (surreal/learner/dqn.py:10-92, model/q_net.py:9-65,
agent/q_agent.py:35-53, utils/schedule.py:34-99) with the stand-ins the reference lacks filled in as DESIGN.md §4 pins
them: openai-baselines' Huber with delta 1, clone / copy_from as parameter copies, clip_grad_norm as
torch.nn.utils.clip_grad_norm_.  Layers are (weight [out, in], bias [out]) pairs in torch.nn.Linear's convention."""
import numpy as np
import torch

from .philox import philox4x32_10


def huber(x):
    """0.5 x^2 for |x| < 1, |x| - 0.5 otherwise (openai-baselines huber_loss, delta = 1)."""
    return torch.where(x.abs() < 1.0, 0.5 * x * x, x.abs() - 0.5)


def tower(x, layers):
    """Linear-ReLU-...-Linear."""
    h = x
    for i, (w, b) in enumerate(layers):
        h = h @ w.t() + b
        if i + 1 < len(layers):
            h = torch.relu(h)
    return h


def combine(a, v):
    """Q = (A - mean_j A) + V (q_net.py:52-59), or A without a state tower."""
    return a if v is None else (a - a.mean(1, keepdim=True)) + v


def q_values(x, action_layers, state_layers=None):
    return combine(tower(x, action_layers), tower(x, state_layers) if state_layers is not None else None)


def td_loss(qa, qv, ta, tv, oa, ov, actions, rewards, dones, weights, gamma):
    """dqn.py:44-69 from the towers' outputs: (loss, td [B])."""
    q = combine(qa, qv)
    a = actions.long().view(-1, 1)
    q_t = q.gather(1, a)
    q_tp1 = combine(ta, tv).detach()
    if oa is not None:
        best = combine(oa, ov).detach().max(1, keepdim=True)[1]
        q_best = q_tp1.gather(1, best)
    else:
        q_best = q_tp1.max(1, keepdim=True)[0]
    q_best = (1.0 - dones.view(-1, 1)) * q_best
    y = rewards.view(-1, 1) + gamma * q_best
    td = q_t - y
    w = torch.ones_like(td) if weights is None else weights.view(-1, 1)
    return torch.mean(w * huber(td)), td.view(-1)


class OracleDQN:
    """DQNLearner._optimize + _run_optimizer + the sample-counted target copy, in float64."""

    def __init__(self, action_layers, state_layers, lr, gamma, double_q, target_period, grad_norm_clipping=10.0,
                 adam_eps=1e-4, target_action_layers=None, target_state_layers=None):
        """``target_*_layers``: the target network's own weights (default: a copy of the online ones, dqn.py:17)."""
        p = lambda layers: [(w.double().clone().requires_grad_(), b.double().clone().requires_grad_())  # noqa: E731
                            for w, b in layers]
        self.a = p(action_layers)
        self.v = p(state_layers) if state_layers is not None else None
        self.params = [t for wb in self.a + (self.v or []) for t in wb]
        c = lambda layers: [(w.detach().double().clone(), b.detach().double().clone()) for w, b in layers]  # noqa: E731
        self.ta = c(target_action_layers if target_action_layers is not None else self.a)
        self.tv = None
        if self.v is not None:
            self.tv = c(target_state_layers if target_state_layers is not None else self.v)
        self.opt = torch.optim.Adam(self.params, lr=lr, eps=adam_eps)
        self.gamma, self.double_q, self.period, self.clip = gamma, double_q, int(target_period), grad_norm_clipping
        self.samples = 0

    def update(self, obs, actions, rewards, obs_next, dones, weights=None):
        """-> dict(loss, td_error, q_value, td [B])."""
        d = lambda t: torch.as_tensor(np.asarray(t), dtype=torch.float64)  # noqa: E731
        obs, obs_next, actions, rewards, dones = d(obs), d(obs_next), d(actions), d(rewards), d(dones)
        w = d(weights) if weights is not None else None
        qa = tower(obs, self.a)
        qv = tower(obs, self.v) if self.v is not None else None
        ta = tower(obs_next, self.ta)
        tv = tower(obs_next, self.tv) if self.tv is not None else None
        oa = ov = None
        if self.double_q:
            with torch.no_grad():
                oa = tower(obs_next, self.a)
                ov = tower(obs_next, self.v) if self.v is not None else None
        loss, td = td_loss(qa, qv, ta, tv, oa, ov, actions, rewards, dones, w, self.gamma)
        q = combine(qa, qv).gather(1, actions.long().view(-1, 1))
        self.opt.zero_grad()
        loss.backward()
        if self.clip is not None:
            torch.nn.utils.clip_grad_norm_(self.params, self.clip)
        self.opt.step()
        B = obs.shape[0]
        if (self.samples + B) // self.period > self.samples // self.period:      # PeriodicTracker(period), += B
            self.ta = [(w_.detach().clone(), b_.detach().clone()) for w_, b_ in self.a]
            if self.v is not None:
                self.tv = [(w_.detach().clone(), b_.detach().clone()) for w_, b_ in self.v]
        self.samples += B
        return {'loss': float(loss.detach()), 'td_error': float(td.abs().mean()), 'q_value': float(q.mean()),
                'td': td.detach()}


def act_draws(seed, counter, actors, n_actions):
    """(u [len], uniform action [len]) of sb200_dqn_act_f32: Philox4x32-10 keyed (seed, counter, actor); u = x / 2^32,
    action = floor(y * n / 2^32)."""
    ids = np.asarray(actors, dtype=np.uint64)
    x, y, _, _ = philox4x32_10(np.uint64(seed), np.uint64(counter), ids)
    u = x.astype(np.float64) * 2.0 ** -32
    a = (y.astype(np.uint64) * np.uint64(n_actions)) >> np.uint64(32)
    return u, a.astype(np.int64)


def act(q, eps, seed, counter):
    """QAgent.act for a batch of actors on Q rows [N, n] (float64 numpy): greedy argmax (first index among ties) unless
    u < eps, then the uniform draw."""
    q = np.asarray(q)
    N, n = q.shape
    u, ra = act_draws(seed, counter, np.arange(N), n)
    greedy = q.argmax(1)
    return np.where(u < eps, ra, greedy)
