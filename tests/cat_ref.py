"""TEST INFRASTRUCTURE -- the categorical PPO policy of a discrete action space in float64: its distribution functions,
its Philox draw, and PPO learners that run it through the oracle's learn() flows (oracle/ppo.py, ppo_rnn.py,
ppo_pixel.py) for the MLP, LSTM and CNN stems.

The reference names a discrete action_spec but has no categorical distribution; these functions define the semantics
the device kernels implement (surreal_b200/csrc/ppo_cat.cu).  ``prob`` rows are ``[p(K) | log p(K)]``; actions are
one-hot rows [K].  Each function takes the same (a, prob, d) / (prob0, prob1, d) arguments as its DiagGauss counterpart
in oracle/pd.py.
"""
import numpy as np
import torch

from oracle import nets
from oracle.philox import philox4x32_10
from oracle.ppo import OraclePPOLearner
from oracle.ppo_pixel import OraclePPOLearnerPixel
from oracle.ppo_rnn import OraclePPOLearnerRNN

F64 = torch.float64


def _split(prob, d):
    prob = prob.reshape(-1, 2 * d)
    return prob[:, :d], prob[:, d:]


def cat_prob(logits):
    """logits [rows, K] -> pd rows [rows, 2K] = [p | log p] from a max-subtracted log-softmax (differentiable)."""
    z = logits - logits.max(dim=1, keepdim=True)[0].detach()
    logp = z - z.exp().sum(dim=1, keepdim=True).log()
    return torch.cat([logp.exp(), logp], dim=1)


def cat_loglikelihood(a, prob, d):
    """log p_a of the one-hot rows ``a`` -> shape [rows, 1]."""
    return (a.reshape(-1, d) * _split(prob, d)[1]).sum(dim=1, keepdim=True)


def cat_likelihood(a, prob, d):
    """max(p_a, 1e-5) -> shape [rows, 1], the clamp of DiagGauss.likelihood (its gradient is zero where it binds)."""
    return torch.clamp((a.reshape(-1, d) * _split(prob, d)[0]).sum(dim=1, keepdim=True), min=1e-5)


def cat_kl(prob0, prob1, d):
    """KL(p0 || p1) = sum_j p0_j (log p0_j - log p1_j) -> shape [rows]; a term with p0_j = 0 contributes 0."""
    p0, l0 = _split(prob0, d)
    _, l1 = _split(prob1, d)
    return torch.where(p0 > 0, p0 * (l0 - l1), torch.zeros_like(p0)).sum(dim=1)


def cat_entropy(prob, d):
    """-sum_j p_j log p_j -> shape [rows]; a term with p_j = 0 contributes 0."""
    p, lp = _split(prob, d)
    return -torch.where(p > 0, p * lp, torch.zeros_like(p)).sum(dim=1)


def cat_sample(prob_np, d, u):
    """Inverse CDF with one uniform per row (``u`` [rows], agent_uniform): the first j with u < c_j, c_j the running sum
    of p_0..p_j in index order, or d - 1 when u is not below c_{d-1} -> int64 [rows]."""
    c = np.cumsum(np.asarray(prob_np, dtype=np.float64).reshape(-1, 2 * d)[:, :d], axis=1)
    below = np.asarray(u, dtype=np.float64)[:, None] < c
    return np.where(below.any(axis=1), below.argmax(axis=1), d - 1).astype(np.int64)


def cat_maxprob(prob_np, d):
    """argmax_j p_j, the lowest index among ties -> int64 [rows]."""
    return np.asarray(prob_np).reshape(-1, 2 * d)[:, :d].argmax(axis=1).astype(np.int64)


def agent_uniform(agent_seed, step, actor_ids):
    """The uniform of the categorical PPOAgent.act draw at global step `step` -> [len(ids)] float64 (exact): the first
    word x of oracle.philox's Philox4x32-10 keyed as agent_eps keys its first group (agent seed, step, actor << 16),
    u = (x >> 8) / 2^24."""
    ids = np.asarray(actor_ids, dtype=np.uint64)
    x, _, _, _ = philox4x32_10(np.uint64(agent_seed), np.uint64(step), ids << np.uint64(16))
    return (x >> np.uint32(8)).astype(np.float64) * 2.0 ** -24


# -- learners ----------------------------------------------------------------------------------------------------------
def _f64(layers):
    return [(w.to(F64), b.to(F64)) for w, b in layers]


class _Categorical:
    """The categorical policy on top of an oracle learner, in float64: the actor's last layer outputs the K logits, pd rows
    are cat_prob of them, and the losses, KL early stop and closing statistics use the cat_* functions.  The base class
    is built with a zero log_var that takes no part in the policy (it is not a parameter of the optimisers).  _rows
    selects the update rows of a window batch (step 0, or the first eff_len steps in RNN mode)."""

    def _cat_setup(self, stem_params):
        c, stem = self.c, list(stem_params)                           # both optimisers train the shared stems
        self.actor_params = [t for wb in self.actor for t in wb] + stem
        self.critic_params = [t for wb in self.critic for t in wb] + stem
        self.actor_optim = torch.optim.Adam(self.actor_params, lr=c['lr_actor'])
        self.critic_optim = torch.optim.Adam(self.critic_params, lr=c['lr_critic'])

    def _head(self, x, ref=False):
        return cat_prob(nets.mlp_trunk(x, self.ref_actor if ref else self.actor))

    def preprocess(self, batch):                                      # ppo.py:420-484 in float64
        t = lambda k: torch.tensor(np.asarray(batch[k]), dtype=F64)  # noqa: E731
        obs, obs_next, actions = t('obs'), t('obs_next'), t('actions')
        rewards = t('rewards') * self.c['reward_scale']
        if self.rfilter is not None:
            normed = self.rfilter.forward(rewards)
            self.rfilter.update(rewards)
            rewards = normed
        return obs, obs_next, actions, rewards, t('dones'), t('pd')

    def _clip_loss(self, obs, actions, adv, behave_pol):              # ppo.py:194-225
        learn_pol = self.forward_actor(obs)
        ratio = cat_likelihood(actions, learn_pol, self.A) / cat_likelihood(actions, behave_pol, self.A)
        clipped = torch.clamp(ratio, 1 - self.clip_epsilon, 1 + self.clip_epsilon)
        surr = -ratio * adv.reshape(-1, 1)
        csurr = -clipped * adv.reshape(-1, 1)
        loss = torch.cat([surr, csurr], 1).max(1)[0].mean()
        stats = {'_surr_loss': surr.mean().item(), '_clip_surr_loss': loss.item(),
                 '_entropy': cat_entropy(learn_pol, self.A).mean().item(), '_clip_epsilon': self.clip_epsilon}
        return loss, stats

    def _adapt_loss(self, obs, actions, adv, behave_pol, ref_pol):    # ppo.py:250-285
        learn_pol = self.forward_actor(obs)
        prob_behave = cat_likelihood(actions, behave_pol, self.A)
        prob_learn = cat_likelihood(actions, learn_pol, self.A)
        kl = cat_kl(ref_pol, learn_pol, self.A).mean()
        surr = -(adv.reshape(-1, 1) * (prob_learn / torch.clamp(prob_behave, min=1e-2))).mean()
        loss = surr + self.beta * kl
        if kl.item() - 2.0 * self.c['kl_target'] > 0:
            loss = loss + self.c['kl_cutoff_coeff'] * (kl - 2.0 * self.c['kl_target']).pow(2)
        stats = {'_kl_loss_adapt': loss.item(), '_surr_loss': surr.item(), '_pol_kl': kl.item(),
                 '_entropy': cat_entropy(learn_pol, self.A).mean().item(), '_beta': self.beta}
        return loss, stats

    def _set_cells(self, batch):
        pass

    def _rows(self, t):
        return t[:, 0].contiguous()

    def learn(self, batch):                                           # ppo.py:588-613 + 487-586
        self.current_iteration += 1
        obs, obs_next, actions, rewards, dones, pds = self.preprocess(batch)
        self._set_cells(batch)
        adv, ret = self.gae_and_return(obs, obs_next, rewards, dones)
        adv, ret = adv.detach(), ret.detach()
        self.last_adv, self.last_ret = adv, ret
        behave_pol, acts, obs_u = self._rows(pds), self._rows(actions), self._rows(obs)
        ref_pol = self.forward_actor(obs_u, ref=True).detach()
        n_ep = 0
        for _ in range(self.c['epoch_policy']):
            stats = self._policy_update(obs_u, acts, adv, behave_pol, ref_pol)
            n_ep += 1
            curr_pol = self.forward_actor(obs_u).detach()
            klv = cat_kl(ref_pol, curr_pol, self.A).mean()
            stats['_pol_kl'] = klv.item()
            if klv.item() > self.c['kl_target'] * 4:
                break
        self.n_policy_epochs.append(n_ep)
        self.kl_record.append(stats['_pol_kl'])
        for _ in range(self.c['epoch_baseline']):
            bstats = self._value_update(obs_u, ret)
        stats.update(bstats)
        behave_lik = cat_likelihood(acts, behave_pol, self.A)
        curr_lik = cat_likelihood(acts, curr_pol, self.A)
        stats['_avg_return_targ'] = ret.mean().item()                 # no log_var: no _avg_log_sig
        stats['_avg_behave_likelihood'] = behave_lik.mean().item()
        stats['_avg_is_weight'] = (curr_lik / (behave_lik + 1e-4)).mean().item()
        stats['_ref_behave_diff'] = cat_kl(ref_pol, behave_pol, self.A).mean().item()
        stats['_lr'] = self.actor_optim.param_groups[0]['lr']
        if self.zf is not None:
            self.zf.update(obs_u)                                     # ppo.py:578-579 (AFTER the updates)
            stats['obs_running_mean'] = float(np.mean(self.zf.running_mean()))
            stats['obs_running_square'] = float(np.mean(self.zf.running_square()))
            stats['obs_running_std'] = float(np.mean(self.zf.running_std()))
        if self.rfilter is not None:
            stats['reward_mean'] = self.rfilter.reward_mean()
        self.exp_counter += self.batch_size
        return stats


class CatOraclePPOLearner(_Categorical, OraclePPOLearner):
    """MLP stem (oracle/ppo.py)."""

    def __init__(self, actor_layers, critic_layers, zfilter, n_actions, n_step, batch_size, **cfg):
        super().__init__(_f64(actor_layers), torch.zeros(1, n_actions, dtype=F64), _f64(critic_layers), zfilter,
                         n_actions, n_step, batch_size, **cfg)
        self._cat_setup([])

    def forward_actor(self, obs, ref=False):
        zf = self.ref_zf if ref else self.zf
        return self._head(zf.forward(obs) if zf is not None else obs, ref)


class CatOraclePPOLearnerRNN(_Categorical, OraclePPOLearnerRNN):
    """LSTM stem (oracle/ppo_rnn.py): cells from the batch's h0 / c0 [B, layers, H]."""

    def __init__(self, actor_layers, critic_layers, zfilter, lstm_state, n_actions, n_step, batch_size, horizon,
                 rnn_hidden, rnn_layer=1, **cfg):
        super().__init__(_f64(actor_layers), torch.zeros(1, n_actions, dtype=F64), _f64(critic_layers), zfilter,
                         lstm_state, n_actions, n_step, batch_size, horizon, rnn_hidden, rnn_layer, **cfg)
        self.rnn.to(F64)
        self.ref_rnn.to(F64)
        self._cat_setup(self.rnn.parameters())

    def forward_actor(self, obs, ref=False):
        zf = self.ref_zf if ref else self.zf
        x = zf.forward(obs) if zf is not None else obs
        feat, _ = (self.ref_rnn if ref else self.rnn)(x, self.cells)
        shp = feat.shape
        return self._head(feat.contiguous().view(-1, shp[2]), ref).view(shp[0], shp[1], -1)

    def _set_cells(self, batch):
        cells = [torch.tensor(np.asarray(batch[k]), dtype=F64).transpose(0, 1).contiguous() for k in ('h0', 'c0')]
        self.cells = tuple(cells)

    def _rows(self, t):
        return t[:, :self.n_step - self.horizon + 1].contiguous()


class CatOraclePPOLearnerPixel(_Categorical, OraclePPOLearnerPixel):
    """CNN stem (oracle/ppo_pixel.py)."""

    def __init__(self, actor_layers, critic_layers, conv_layers, strides, fc_layer, n_actions, n_step, batch_size, **cfg):
        super().__init__(_f64(actor_layers), torch.zeros(1, n_actions, dtype=F64), _f64(critic_layers),
                         _f64(conv_layers), strides, _f64([fc_layer])[0], n_actions, n_step, batch_size, **cfg)
        self._cat_setup([t for wb in self.conv for t in wb] + list(self.fc))

    def forward_actor(self, obs, ref=False):
        return self._head(self.stem(obs, ref), ref)

