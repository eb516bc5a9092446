"""DDPGLearner: drop-in for surreal/learner/ddpg.py:12-440 (low-dim observations) running on hand-written kernels:
target nets -> Bellman target -> critic MSE step -> actor step THROUGH the updated critic -> target update.
Statistics names and the order of operations follow ddpg.py:244-352, including the TD3 options
(``use_double_critic``: second critic + target, y = min(y, y2); ``use_action_regularization``: clipped noise on the
target action -- added, as in the reference, only AFTER Q'_1 was evaluated, so it reaches critic 2 alone)."""
import torch

from .. import _lib, ops
from .._lib import check
from .. import utils as U
from ..model.ddpg_net import DDPGModel
from ..ops import _ptr
from ..session import ConfigError
from .aggregator import SSARAggregator
from .off_policy import OffPolicyLearner

DS = dict(ACTOR_LOSS=0, CRITIC_LOSS=1, ACTION_NORM=2, REWARDS=3, Q_TARGET=4, Q_POLICY=5, ABSMAX=6, TD_ERROR=7,
          IS_WEIGHT=8)


class DDPGLearner(OffPolicyLearner):
    bad_action_message = 'actions outside [-1, 1] (ddpg.py:261-262)'

    def __init__(self, learner_config, env_config, session_config):
        super().__init__(learner_config, env_config, session_config)
        if not torch.cuda.is_available():
            raise RuntimeError('surreal_b200.DDPGLearner needs a CUDA device (there is no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.current_iteration = 0
        lc = self.learner_config
        self.batch_size = lc.replay.batch_size
        self.discount_factor = lc.algo.gamma
        self.n_step = lc.algo.n_step
        self.is_pixel_input = self.env_config.pixel_input
        self.use_layernorm = lc.model.use_layernorm
        self.use_double_critic = lc.algo.network.use_double_critic
        self.use_action_regularization = lc.algo.network.use_action_regularization
        self._num_gpus = 1
        cfg = lc.algo.network.target_update                                 # ddpg.py:403-428
        self.target_update_type = cfg.type
        if cfg.type == 'soft':
            self.target_update_tau = cfg.tau
        elif cfg.type == 'hard':
            self.target_update_counter = 0
            self.target_update_interval = cfg.interval
        else:
            raise ConfigError('Unsupported ddpg update type: {}'.format(cfg.type))
        net = lc.algo.network
        self.clip_actor_gradient = net.clip_actor_gradient
        self.actor_gradient_clip_value = net.actor_gradient_value_clip if self.clip_actor_gradient else 0.0
        self.clip_critic_gradient = net.clip_critic_gradient
        self.critic_gradient_clip_value = net.critic_gradient_value_clip if self.clip_critic_gradient else 0.0
        self.action_dim = self.env_config.action_spec.dim[0]
        mk = dict(obs_spec=self.env_config.obs_spec, action_dim=self.action_dim, use_layernorm=self.use_layernorm,
                  actor_fc_hidden_sizes=lc.model.actor_fc_hidden_sizes,
                  critic_fc_hidden_sizes=lc.model.critic_fc_hidden_sizes, device=self.device)
        self.model = DDPGModel(**mk)
        self.model_target = DDPGModel(**mk)
        B, A = self.batch_size, self.action_dim
        D = self.model.input_dim
        self.low_dim = D
        self.critic_optim = ops.MlpTrainer(self.model.critic, B, net.lr_critic,
                                           clip_mode=2 if self.clip_critic_gradient else 0,
                                           clip_value=self.critic_gradient_clip_value,
                                           weight_decay=net.critic_regularization)
        self.actor_optim = ops.MlpTrainer(self.model.actor, B, net.lr_actor,
                                          clip_mode=2 if self.clip_actor_gradient else 0,
                                          clip_value=self.actor_gradient_clip_value,
                                          weight_decay=net.actor_regularization)
        self.model2 = self.model_target2 = self.critic_optim2 = None
        if self.use_double_critic:                                           # ddpg.py:118-143,157-162
            self.model2 = DDPGModel(critic_only=True, **mk)
            self.model_target2 = DDPGModel(critic_only=True, **mk)
            self.critic_optim2 = ops.MlpTrainer(self.model2.critic, B, net.lr_critic,
                                                clip_mode=2 if self.clip_critic_gradient else 0,
                                                clip_value=self.critic_gradient_clip_value,
                                                weight_decay=net.critic_regularization)
            self.model_target2.critic.params.copy_(self.model2.critic.params)
        self.aggregator = SSARAggregator(self.env_config.obs_spec, self.env_config.action_spec)
        self.model_target.actor.params.copy_(self.model.actor.params)        # hard_update (ddpg.py:174-175)
        self.model_target.critic.params.copy_(self.model.critic.params)
        self.total_learn_time = U.TimeRecorder()
        self.forward_time = U.TimeRecorder()
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)  # noqa: E731
        self._pi_t, self._q_t, self._y = f(B, A), f(B, 1), f(B)
        self._dA = f(B, ops._ru(A, 4))
        self._pi_t2, self._q_t2 = f(B, A), f(B, 1)
        self.policy_noise, self.noise_clip = 0.2, 0.5           # hard-coded in the reference (ddpg.py:269-270)
        self._noise_draws = None                                # tests: injected N(0,1) draws [B, A], see setter below
        self._td3_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._td3_seed = 77
        self._ws = torch.zeros(_lib.lib().sb200_ddpg_workspace_bytes(B), dtype=torch.uint8, device=self.device)
        # prioritized replay: a batch with importance weights takes the weighted critic loss (dqn.py:148-168), whose
        # rows also give the sampled records' new priorities |q1 - y| + eps (critic 1's TD error, before the step)
        rc = lc.replay
        self.priority_eps = float(rc.priority_eps) if 'priority_eps' in rc else 1e-6
        # the target kernel raises the workspace's bad-action flag when max|a| > 1: every optimiser / target kernel of
        # the call then no-ops, so the AssertionError leaves the learner exactly as the reference's pre-update assert does
        hard = self.target_update_type == 'hard'
        self._init_off_policy(D, A, 32, self._ws, int(_lib.lib().sb200_ddpg_bad_action_offset()),
                              tau=None if hard else self.target_update_tau,
                              counter='target_update_counter' if hard else None,
                              period=self.target_update_interval if hard else 1)
        self._stats = self._stats_block[0:16]
        self._stats2 = self._stats_block[16:32]                # critic 2's loss / Q (critic_loss is overwritten by it)

    # ------------------------------------------------------------------------------------------------
    @property
    def policy_noise_draws(self):
        return self._noise_draws

    @policy_noise_draws.setter
    def policy_noise_draws(self, draws):
        """Inject the N(0,1) draws of the TD3 target-action noise (parity tests).  They live in ONE persistent buffer,
        so a captured graph keeps reading the right address; must be set before the first learn() (a graph captured
        with Philox noise keeps using Philox)."""
        if self._noise_draws is None:
            self._noise_draws = torch.zeros(self.batch_size, self.action_dim, dtype=torch.float32, device=self.device)
        self._noise_draws.copy_(torch.as_tensor(draws, dtype=torch.float32).reshape(self.batch_size, self.action_dim))

    def _critic_loss(self, trainer, q, stats, weights, prio):
        L, st, B = _lib.lib(), ops._stream(), self.batch_size
        d = trainer.d[-1]
        if weights is None:
            check(L.sb200_ddpg_critic_loss_f32(_ptr(q), q.stride(0), _ptr(self._y), B, _ptr(d), d.stride(0), _ptr(stats),
                                               _ptr(self._ws), st), 'sb200_ddpg_critic_loss_f32')
        else:
            check(L.sb200_ddpg_critic_loss_weighted_f32(_ptr(q), q.stride(0), _ptr(self._y), B, _ptr(weights), _ptr(d),
                                                        d.stride(0), _ptr(prio), self.priority_eps, _ptr(stats),
                                                        _ptr(self._ws), st), 'sb200_ddpg_critic_loss_weighted_f32')

    def _optimize_device(self, weights):
        """ddpg.py:244-333 as one fixed launch sequence (CUDA-graph body; no host round trip inside).  ``weights``
        (device [B, 1]): importance weights of a prioritized batch; both critic losses are weighted and critic 1's rows
        leave the new priorities |q1 - y| + priority_eps in ``td_priorities``."""
        L = _lib.lib()
        B, A = self.batch_size, self.action_dim
        mt, st = self.model_target, ops._stream()
        b = self._own
        obs, obs_next, actions, rewards, dones = b['obs'], b['obs_next'], b['actions'], b['rewards'], b['dones']
        ops.mlp_forward(mt.actor, obs_next, out=self._pi_t)                              # ddpg.py:266
        ops.mlp_forward(mt.critic, obs_next, aux=self._pi_t, out=self._q_t)
        pi2 = self._pi_t
        if self.use_action_regularization:                                               # ddpg.py:267-278
            check(L.sb200_ddpg_smooth_action_f32(_ptr(self._pi_t), A, _ptr(self._noise_draws), B, A,
                                                 self.policy_noise, self.noise_clip, self._td3_seed,
                                                 _ptr(self._td3_counter), _ptr(self._pi_t2), A, st),
                  'sb200_ddpg_smooth_action_f32')
            self._td3_counter += 1
            pi2 = self._pi_t2
        disc = float(pow(self.discount_factor, self.n_step))
        if self.use_double_critic:                                                       # ddpg.py:280-283
            ops.mlp_forward(self.model_target2.critic, obs_next, aux=pi2, out=self._q_t2)
            check(L.sb200_ddpg_target2_f32(_ptr(rewards), _ptr(self._q_t), 1, _ptr(self._q_t2), 1, _ptr(dones),
                                           _ptr(actions), A, B, A, disc, _ptr(self._y), _ptr(self._stats),
                                           _ptr(self._ws), st), 'sb200_ddpg_target2_f32')
        else:
            check(L.sb200_ddpg_target_f32(_ptr(rewards), _ptr(self._q_t), 1, _ptr(dones), _ptr(actions), A, B, A,
                                          disc, _ptr(self._y), _ptr(self._stats), _ptr(self._ws), st),
                  'sb200_ddpg_target_f32')
        stop = self._latch_bad_action()
        ct = self.critic_optim
        q = ct.forward(obs, aux=actions)                                                # Q(s_t, a_t)
        self._critic_loss(ct, q, self._stats, weights, self._prio)
        ct.backward()
        ct.step(stop_flag=stop)
        if self.use_double_critic:                                                       # ddpg.py:298-303,311-321
            c2 = self.critic_optim2
            q2 = c2.forward(obs, aux=actions)
            self._critic_loss(c2, q2, self._stats2, weights, None)
            c2.backward()
            c2.step(stop_flag=stop)
        at = self.actor_optim
        a_pi = at.forward(obs)
        q_pi = ct.forward(obs, aux=at.h[-1])                  # through the UPDATED critic (ddpg.py:324-327)
        check(L.sb200_ddpg_actor_seed_f32(_ptr(q_pi), q_pi.stride(0), B, _ptr(ct.d[-1]), ct.d[-1].stride(0),
                                          _ptr(self._stats), _ptr(self._ws), st), 'sb200_ddpg_actor_seed_f32')
        ct.backward_inputs(stop_layer=1)
        ct.grad_wrt_aux(1, self._dA)
        check(L.sb200_tanh_bwd_f32(_ptr(self._dA), self._dA.stride(0), _ptr(a_pi), a_pi.stride(0), B, A,
                                   _ptr(at.d[-1]), at.d[-1].stride(0), st), 'sb200_tanh_bwd_f32')
        at.backward()
        at.step(stop_flag=stop)

    def _target_pairs(self):
        pairs = [(self.model_target.actor, self.model.actor), (self.model_target.critic, self.model.critic)]
        if self.use_double_critic:
            pairs.append((self.model_target2.critic, self.model2.critic))
        return pairs

    def _statistics(self, s, weighted):
        stats = {'actor_loss': float(s[DS['ACTOR_LOSS']]), 'critic_loss': float(s[DS['CRITIC_LOSS']]),
                 'action_norm': float(s[DS['ACTION_NORM']]), 'rewards': float(s[DS['REWARDS']]),
                 'Q_target': float(s[DS['Q_TARGET']]), 'Q_policy': float(s[DS['Q_POLICY']]),
                 'performance/forward_time': self.forward_time.avg}
        # (the reference's critic_update_time / actor_update_time split does not exist here: the whole update is one
        #  CUDA graph; performance/forward_time covers it)
        if self.use_double_critic:                               # ddpg.py:316,345-346: critic_loss is critic 2's
            s2 = s[16:32]
            stats['critic_loss'] = float(s2[DS['CRITIC_LOSS']])
            stats['Q_policy2'] = float(s2[DS['Q_POLICY']])
        if weighted:                                             # prioritized replay only (dqn.py's td_error)
            stats['td_error'] = float(s[DS['TD_ERROR']])
            stats['avg_is_weight'] = float(s[DS['IS_WEIGHT']])
        return stats

    def module_dict(self):
        return {'ddpg': self.model}

    def checkpoint_attributes(self):
        attrs = ['current_iteration', 'model', 'model_target']
        if self.use_double_critic:
            attrs += ['model2', 'model_target2']
        ck = self.session_config.checkpoint.learner
        if 'include_optimizer' in ck and ck.include_optimizer:     # extension (off by default): bit-identical continuation
            attrs += ['actor_optim', 'critic_optim', 'target_update_counter'] if self.target_update_type == 'hard' \
                else ['actor_optim', 'critic_optim']
            if self.use_double_critic:
                attrs += ['critic_optim2']
        return attrs

    def _prefetcher_preprocess(self, batch):
        if isinstance(batch, dict):
            return batch
        return self.aggregator.aggregate(batch)
