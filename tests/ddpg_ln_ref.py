"""TEST INFRASTRUCTURE -- CPU restatement of the LayerNorm DDPG networks (``model.use_layernorm``,
surreal/model/model_builders/builders.py:35-84) and of what consumes them: DDPGLearner._optimize (ddpg.py:244-428),
DDPGAgent.act (ddpg_agent.py:155-184) and the flat per-actor image layout of parameter noise.  It extends the oracle of
oracle/ (which restates the plain networks) without changing it.

A network is a list of per-layer tuples: (W [out, in], b [out]) for a plain layer, (W, b, gain, bias) for a hidden layer
followed by its LayerNorm: Linear -> ReLU -> LayerNorm.  The reference's torchx ``LayerNorm(1)`` is torch.nn.LayerNorm
over the last dimension: eps 1e-5, elementwise affine, biased variance (tests/golden/_ref_harness.py)."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.param_noise import _ru

LAYERNORM_EPS = 1e-5


# -- networks ----------------------------------------------------------------------------------------------------------
def params_from_state(sd, prefix, n_layers, ln_last=False):
    """Entries of a reference state dict ('/' separators) whose Sequential holds Linear, ReLU, LayerNorm per hidden layer:
    Linear at seq/{0,3,6}, LayerNorm at seq/{2,5}.  The last Linear has no LayerNorm unless ``ln_last`` (the critic's
    model_obs, whose only layer is a hidden one)."""
    t = lambda k: torch.tensor(sd['%sseq/%s' % (prefix, k)])  # noqa: E731
    out = []
    for i in range(n_layers):
        e = (t('%d/weight' % (3 * i)), t('%d/bias' % (3 * i)))
        if i + 1 < n_layers or ln_last:
            e += (t('%d/weight' % (3 * i + 2)), t('%d/bias' % (3 * i + 2)))
        out.append(e)
    return out


def actor_layers(sd, prefix='actor/model/'):
    return params_from_state(sd, prefix, 3)


def critic_layers(sd, prefix='critic/'):
    return (params_from_state(sd, prefix + 'model_obs/', 1, ln_last=True) +
            params_from_state(sd, prefix + 'model_concat/', 2))


def hidden(x, entry):
    """Linear -> ReLU [-> LayerNorm when the entry carries (gain, bias)]."""
    h = torch.relu(F.linear(x, entry[0], entry[1]))
    if len(entry) == 4:
        h = F.layer_norm(h, h.shape[-1:], entry[2], entry[3], eps=LAYERNORM_EPS)
    return h


def ddpg_actor(x, layers):
    """ActorNetworkX (builders.py:35-56): hidden layers, tanh output."""
    h = x
    for entry in layers[:-1]:
        h = hidden(h, entry)
    return torch.tanh(F.linear(h, layers[-1][0], layers[-1][1]))


def ddpg_critic(x, act, layers):
    """CriticNetworkX (builders.py:58-84): cat(LN(relu(L0 x)), act) -> relu(L1 .) -> LN -> L2."""
    h = hidden(x, layers[0])
    h = hidden(torch.cat((h, act), 1), layers[1])
    return F.linear(h, layers[2][0], layers[2][1])


# -- agent -------------------------------------------------------------------------------------------------------------
def ddpg_act(obs_row, actor_layers, sigma, unit_noise):
    """ddpg_agent.py:155-184 with NormalActionNoise: clip -> + sigma * unit_noise (float32, in place) -> clip."""
    with torch.no_grad():
        a = ddpg_actor(torch.tensor(obs_row, dtype=torch.float32).unsqueeze(0), actor_layers).numpy()[0]
    a = a.clip(-1, 1)
    a += sigma * np.asarray(unit_noise)
    return a.clip(-1, 1)


def ddpg_act_ou(obs_row, actor_layers, x_prev, sigma, theta, dt, unit_noise):
    """The same with OrnsteinUhlenbeckActionNoise (action_noise.py:22-39): float64 state, mu = 0."""
    with torch.no_grad():
        a = ddpg_actor(torch.tensor(obs_row, dtype=torch.float32).unsqueeze(0), actor_layers).numpy()[0]
    a = a.clip(-1, 1)
    x = np.asarray(x_prev, dtype=np.float64)
    x = x + theta * (0.0 - x) * dt + sigma * np.sqrt(dt) * np.asarray(unit_noise, dtype=np.float64)
    a += x
    return a.clip(-1, 1), x


# -- learner -----------------------------------------------------------------------------------------------------------
class LayerNormDDPGLearner:
    """DDPGLearner._optimize / _target_update (ddpg.py:244-428) on LayerNorm networks; ``critic2`` / ``critic2_t`` switch
    on the TD3 double critic, ``policy_noise`` feeds the action regularisation (added after Q'_1, as the reference)."""

    def __init__(self, actor, critic, actor_t, critic_t, gamma, n_step, lr_actor, lr_critic, clip_actor, actor_clip,
                 clip_critic, critic_clip, target_type, target_interval, tau, critic2=None, critic2_t=None):
        rg = lambda ls: [tuple(t.clone().requires_grad_(True) for t in e) for e in ls]  # noqa: E731
        ng = lambda ls: [tuple(t.clone() for t in e) for e in ls]  # noqa: E731
        flat = lambda ls: [t for e in ls for t in e]  # noqa: E731
        self.actor, self.critic, self.actor_t, self.critic_t = rg(actor), rg(critic), ng(actor_t), ng(critic_t)
        self.gamma, self.n_step = gamma, n_step
        self.clip_actor, self.actor_clip, self.clip_critic, self.critic_clip = clip_actor, actor_clip, clip_critic, critic_clip
        self.target_type, self.target_interval, self.tau, self.target_counter = target_type, target_interval, tau, 0
        self.actor_params, self.critic_params = flat(self.actor), flat(self.critic)
        self.critic_optim = torch.optim.Adam(self.critic_params, lr=lr_critic)
        self.actor_optim = torch.optim.Adam(self.actor_params, lr=lr_actor)
        self.critic2 = self.critic2_t = None
        if critic2 is not None:
            self.critic2, self.critic2_t = rg(critic2), ng(critic2_t)
            self.critic2_params = flat(self.critic2)
            self.critic_optim2 = torch.optim.Adam(self.critic2_params, lr=lr_critic)

    def _critic_step(self, params, optim, q, y):
        for p in params:
            p.grad = None
        loss = nn.MSELoss()(q, y)
        loss.backward()
        if self.clip_critic:
            nn.utils.clip_grad_value_(params, self.critic_clip)
        optim.step()
        return loss

    def optimize(self, obs, actions, rewards, obs_next, dones, policy_noise=None):
        obs, obs_next, actions = (torch.tensor(v, dtype=torch.float32) for v in (obs, obs_next, actions))
        rewards, dones = torch.tensor(rewards, dtype=torch.float32), torch.tensor(dones, dtype=torch.float32)
        with torch.no_grad():
            pol_t = ddpg_actor(obs_next, self.actor_t)
            q_t = ddpg_critic(obs_next, pol_t, self.critic_t)
            if policy_noise is not None:
                pol_t = (pol_t + torch.tensor(np.clip(np.asarray(policy_noise), -0.5, 0.5), dtype=torch.float32)).clamp(-1, 1)
            y = rewards + pow(self.gamma, self.n_step) * q_t * (1.0 - dones)
            if self.critic2 is not None:
                y2 = rewards + pow(self.gamma, self.n_step) * ddpg_critic(obs_next, pol_t, self.critic2_t) * (1.0 - dones)
                y = torch.min(y, y2)
        y_policy = ddpg_critic(obs, actions, self.critic)
        critic_loss = self._critic_step(self.critic_params, self.critic_optim, y_policy, y)
        y_policy2 = None
        if self.critic2 is not None:
            y_policy2 = ddpg_critic(obs, actions, self.critic2)
            critic_loss = self._critic_step(self.critic2_params, self.critic_optim2, y_policy2, y)
        for p in self.actor_params:
            p.grad = None
        actor_loss = -ddpg_critic(obs, ddpg_actor(obs, self.actor), self.critic).mean()
        actor_loss.backward()
        if self.clip_actor:
            nn.utils.clip_grad_value_(self.actor_params, self.actor_clip)
        self.actor_optim.step()
        stats = {'actor_loss': actor_loss.item(), 'critic_loss': critic_loss.item(),
                 'action_norm': actions.norm(2, 1).mean().item(), 'rewards': rewards.mean().item(),
                 'Q_target': y.mean().item(), 'Q_policy': y_policy.mean().item()}
        if y_policy2 is not None:
            stats['Q_policy2'] = y_policy2.mean().item()
        pairs = list(zip(self.actor_t, self.actor)) + list(zip(self.critic_t, self.critic))
        if self.critic2 is not None:
            pairs += list(zip(self.critic2_t, self.critic2))
        if self.target_type == 'soft':
            for et, e in pairs:
                for tt, t in zip(et, e):
                    tt.mul_(1.0 - self.tau).add_(t.detach(), alpha=self.tau)
        else:
            self.target_counter += 1
            if self.target_counter % self.target_interval == 0:
                for et, e in pairs:
                    for tt, t in zip(et, e):
                        tt.copy_(t.detach())
        return stats


# -- flat per-actor images with LayerNorm (surreal_b200/csrc/param_noise.cu, ops.FlatNet(layernorm=True)) ---------------
def flat_layout(dims):
    """[(w_off, b_off, K, N, ldw, g_off, beta_off)] and the flat size: every hidden layer's LayerNorm gain and bias follow
    its bias, [ldw] each; g_off = beta_off = None after the last layer."""
    lay, off = [], 0
    for l in range(len(dims) - 1):
        K, N = dims[l], dims[l + 1]
        ldw = _ru(N, 4)
        w_off, b_off = off, off + K * ldw
        off += K * ldw + ldw
        g_off = beta_off = None
        if l + 2 < len(dims):
            g_off, beta_off = off, off + ldw
            off += 2 * ldw
        lay.append((w_off, b_off, K, N, ldw, g_off, beta_off))
    return lay, off


def image_stride(dims):
    return _ru(flat_layout(dims)[1], 32)


def to_flat(layers, dims, stride=None, dtype=np.float32):
    """Per-layer tuples -> one flat image (W transposed to [in][ldw], padding zero)."""
    lay, size = flat_layout(dims)
    out = np.zeros(stride if stride is not None else size, dtype=dtype)
    for (w_off, b_off, K, N, ldw, g_off, beta_off), e in zip(lay, layers):
        wt = np.zeros((K, ldw), dtype=dtype)
        wt[:, :N] = np.asarray(e[0]).T
        out[w_off:w_off + K * ldw] = wt.reshape(-1)
        out[b_off:b_off + N] = np.asarray(e[1])
        if g_off is not None:
            out[g_off:g_off + N] = np.asarray(e[2])
            out[beta_off:beta_off + N] = np.asarray(e[3])
    return out


def from_flat(flat, dims):
    lay, _ = flat_layout(dims)
    layers = []
    for (w_off, b_off, K, N, ldw, g_off, beta_off) in lay:
        e = (np.asarray(flat[w_off:w_off + K * ldw]).reshape(K, ldw)[:, :N].T.copy(), np.asarray(flat[b_off:b_off + N]).copy())
        if g_off is not None:
            e += (np.asarray(flat[g_off:g_off + N]).copy(), np.asarray(flat[beta_off:beta_off + N]).copy())
        layers.append(e)
    return layers


def padding_mask(dims, stride):
    """bool [stride]: True at offsets that hold no parameter."""
    L = len(dims) - 1
    ones = [(np.ones((dims[l + 1], dims[l])), np.ones(dims[l + 1])) +
            ((np.ones(dims[l + 1]), np.ones(dims[l + 1])) if l + 1 < L else ()) for l in range(L)]
    return to_flat(ones, dims, stride, dtype=np.float64) == 0.0
