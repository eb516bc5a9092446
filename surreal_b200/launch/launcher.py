"""Component launcher with the reference's surface (surreal/launch/launcher.py:20-440):
``<exe> <component> -- <config flags>``, ``SurrealDefaultLauncher(agent_class, learner_class, replay_class,
session_config, env_config, learner_config)``, ``setup_agent`` / ``setup_learner`` / ``run_replay_worker``.

In the reference every component is its own OS process wired over ZeroMQ by symphony.  Here agents, replay
and learner co-locate in ONE process per GPU, so the launcher's job collapses to constructing the three
plugin objects in the right order and running the engine loop; the pure-plumbing components (ps, tensorplex,
loggerplex, tensorboard, replay load balancer) are accepted and are no-ops."""
import sys
from argparse import ArgumentParser

import numpy as np

from .. import utils as U

_NOOP_COMPONENTS = ('ps', 'tensorplex', 'loggerplex', 'tensorboard', 'replay_loadbalancer')


class Launcher:
    def main(self, argv=None):
        argv = sys.argv[1:] if argv is None else list(argv)
        parser_args, config_args = argv, []
        if '--' in argv:
            i = argv.index('--')
            parser_args, config_args = argv[:i], argv[i + 1:]
        parser = ArgumentParser(description='launch a surreal component')
        parser.add_argument('component_name', type=str, help='which component to launch')
        args = parser.parse_args(parser_args)
        self.config_args = config_args
        self.setup(config_args)
        return self.launch(args.component_name)

    def launch(self, component_name):
        raise NotImplementedError

    def setup(self, args):
        pass


class PipelinedEngine:
    """Actors and learner as two concurrent CUDA streams of ONE process (the single-GPU form of Surreal's asynchronous
    actor / learner processes): while the learner works on batch k, the actors already roll out batch k+1 with the
    weights published after batch k-1 -- exactly the policy lag Surreal's actors run with (docs/ppo.md:16).

      stream A:  [wait pop_k, pub]  rollout_{k+1} .........................  -> roll_{k+1}
      stream L:  [wait roll_k] pop+gather_k -> pop_k | learn_k (CUDA graph) ... publish -> pub

    The rollout is one persistent kernel (or a chain of small kernels) and the learner's persistent kernels want SMs of
    their own: when the rollout runs in one wave on at most half of the SMs, the learner gets the rest as its grid
    budget and learn() runs beside the rollout, so the step time tends to max(rollout, learn) instead of their sum.
    Otherwise the learner's epochs wait for the rollout (before_epochs_hook).  Ordering between the streams is
    carried by events only (FIFO control block: push happens-before pop happens-before next push; parameter
    snapshot: publish happens-before fetch happens-before next publish)."""

    def __init__(self, agent, replay, learner, rollout_steps):
        import torch
        self.torch = torch
        self.agent, self.replay, self.learner, self.T = agent, replay, learner, rollout_steps
        # the actors' stream has the higher priority: when a rollout and a learn() become ready together, the rollout's
        # clusters are placed first and find whole GPCs free (placed after the learner's CTAs they may not fit in one wave)
        self.sA, self.sL = torch.cuda.Stream(priority=-1), torch.cuda.Stream()
        self.ev_roll = self.ev_pop = self.ev_pub = self.ev_fetch = None
        self.iterations = 0
        self.overlap = False
        if hasattr(learner, 'set_sm_budget'):
            n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
            footprint = agent.rollout_footprint() if hasattr(agent, 'rollout_footprint') else 0
            self.overlap = 0 < footprint and 2 * footprint <= n_sm and getattr(learner, 'dp', None) is None
            learner.set_sm_budget(n_sm - footprint if self.overlap else 0)
        if hasattr(learner, 'before_epochs_hook'):
            # learners whose epochs are ONE all-SM persistent kernel take the GPU after the rollout, not beside it
            learner.before_epochs_hook = None if self.overlap else self._wait_rollout
        cur = torch.cuda.current_stream()
        self.sA.wait_stream(cur)
        self.sL.wait_stream(cur)

    def _rollout(self):
        torch = self.torch
        with torch.cuda.stream(self.sA):
            if self.ev_pop is not None:
                self.sA.wait_event(self.ev_pop)
            if self.ev_pub is not None:
                self.sA.wait_event(self.ev_pub)
            self.agent.main_loop(max_steps=self.T)          # parameter fetch (if due) + T batched env steps
            self.ev_fetch = torch.cuda.Event()
            self.ev_fetch.record(self.sA)
            self.ev_roll = torch.cuda.Event()
            self.ev_roll.record(self.sA)

    def _wait_rollout(self):
        """Called by the learner between its head graph and its epochs graph (learner stream current): the rollout that
        was enqueued before this learn() must have finished."""
        if self.ev_roll is not None:
            self.torch.cuda.current_stream().wait_event(self.ev_roll)

    def prime(self):
        """First rollout (nothing to overlap with yet)."""
        self._rollout()

    def step(self):
        """One learner iteration, overlapped with the actors' next rollout.  Returns the learner statistics."""
        torch = self.torch
        L = self.learner
        with torch.cuda.stream(self.sL):
            self.sL.wait_event(self.ev_roll)
            if not self.replay.start_sample_condition():
                raise RuntimeError('replay under-filled: rollout_steps too small for one learner batch')
            data = L.fetch_batch()                           # pop + gather into the learner's buffers
            self.ev_pop = torch.cuda.Event()
            self.ev_pop.record(self.sL)
        self._rollout()                                      # enqueue rollout k+1 BEFORE blocking on learn k
        with torch.cuda.stream(self.sL):
            with L.learn_timer.time():
                stats = L.learn(data)                        # graph replay + one statistics read-back
            if self.ev_fetch is not None:
                self.sL.wait_event(self.ev_fetch)            # the snapshot buffers may still be read by a fetch
            if L.should_publish_parameter():
                L.publish_parameter(L.current_iter, message='batch ' + str(L.current_iter))
            self.ev_pub = torch.cuda.Event()
            self.ev_pub.record(self.sL)
            L.iter_timer.lap()
            L.current_iter += 1
        self.iterations += 1
        return stats

    def drain(self):
        self.torch.cuda.synchronize()


# ReplayEngine defaults: 32 env steps per chunk and one learner update per batched env step (the textbook DDPG ratio).
# Which ratio keeps both streams of an H100 busy has not been measured; pass rollout_steps / updates_per_chunk to tune.
REPLAY_ROLLOUT_STEPS = 32


class ReplayEngine:
    """PipelinedEngine's shape for an off-policy learner on a uniform replay (DDPG): the actors keep inserting into the
    ring while the learner runs K updates per chunk on records it samples ON the device, so neither stream waits for the
    host between two updates.  The single-process form of the reference's free-running actor and learner processes.

      stream A:  [wait view_k, pub]  chunk_{k+1}: T env steps -> ring ..................  -> roll_{k+1}
      stream L:  [wait roll_k] view_k -> view | learn_from_replay(K) (one CUDA graph) | publish -> pub

    view_k (replay.snapshot_view) fixes what the K updates of step k sample from: the ring as chunk k left it, minus the
    W = N * T slots chunk k+1 can overwrite.  Chunk k+1 therefore never writes a slot the learner reads, no record is ever
    torn, and the sampled data do not depend on how the streams interleave: a run equals the one-stream schedule
    (``overlap=False``: chunk, then K updates, in program order) bit for bit.  Against UniformReplay.sample, records
    inserted during the current chunk become eligible one chunk later and the W oldest leave one chunk early.

    Until ``replay.start_sample_condition()`` first holds only the actors run, with one host read of the ring's control
    block per chunk; afterwards the only host synchronisation of a step is the learner's statistics read-back.
    Ordering between the streams is carried by events only (view happens-after chunk k and happens-before chunk k+1;
    publish happens-before fetch happens-before next publish)."""

    def __init__(self, agent, replay, learner, rollout_steps, updates_per_chunk, overlap=True):
        import torch
        from ..session import ConfigError
        self.torch = torch
        self.agent, self.replay, self.learner = agent, replay, learner
        self.T, self.K = int(rollout_steps), int(updates_per_chunk)
        if agent._obs is None:
            agent._obs, _ = agent.env.reset()
        if not agent._device_resident(agent._obs):
            raise ConfigError('ReplayEngine runs device-resident envs only; drive a host env by hand: '
                              'agent.main_loop(T) and, once replay.start_sample_condition() holds, learner.main_loop()')
        self.W = agent.num_envs * self.T                    # most records one chunk can insert
        if replay.memory_size < 2 * self.W:
            raise ConfigError('replay.memory_size {} is less than two chunks of inserts (2 x {} actors x {} steps): the '
                              'sampling view would be empty'.format(replay.memory_size, agent.num_envs, self.T))
        if self.T < 1 or self.K < 1 or replay.learner_config.replay.sampling_start_size < 0:
            raise ConfigError('rollout_steps and updates_per_chunk must be >= 1 and sampling_start_size >= 0')
        self.sA = torch.cuda.Stream(priority=-1)
        self.sL = torch.cuda.Stream() if overlap else self.sA
        self.ev_roll = self.ev_view = self.ev_pub = self.ev_fetch = None
        self.iterations = 0
        self.started = False                                 # the ring has held more than sampling_start_size records
        cur = torch.cuda.current_stream()
        self.sA.wait_stream(cur)
        self.sL.wait_stream(cur)

    def _rollout(self):
        torch = self.torch
        with torch.cuda.stream(self.sA):
            if self.ev_view is not None:
                self.sA.wait_event(self.ev_view)
            if self.ev_pub is not None:
                self.sA.wait_event(self.ev_pub)
            self.agent.main_loop(max_steps=self.T)          # parameter fetch (if due) + T batched env steps
            self.ev_fetch = torch.cuda.Event()
            self.ev_fetch.record(self.sA)
            self.ev_roll = torch.cuda.Event()
            self.ev_roll.record(self.sA)

    def prime(self):
        """First chunk (nothing to overlap with yet)."""
        self._rollout()

    def step(self):
        """One chunk of the actors beside K learner updates on the previous chunks' records.  Returns the learner
        statistics, or None while the ring is still filling."""
        torch = self.torch
        L = self.learner
        if not self.started:
            with torch.cuda.stream(self.sA):
                self.replay.mark_device_inserts()            # a replayed chunk graph inserts without telling the host
                self.started = self.replay.start_sample_condition()     # host read, after the last chunk
            if not self.started:
                self._rollout()
                self.iterations += 1
                return None
        with torch.cuda.stream(self.sL):
            self.sL.wait_event(self.ev_roll)
            self.replay.snapshot_view(reserve=self.W)
            self.ev_view = torch.cuda.Event()
            self.ev_view.record(self.sL)
        self._rollout()                                      # enqueue chunk k+1 BEFORE blocking on the read-back
        with torch.cuda.stream(self.sL):
            with L.learn_timer.time():
                stats = L.learn_from_replay(self.replay, self.K)
            self.sL.wait_event(self.ev_fetch)                # the snapshot buffers may still be read by a fetch
            if L.should_publish_parameter():
                L.publish_parameter(L.current_iter, message='batch ' + str(L.current_iter))
            self.ev_pub = torch.cuda.Event()
            self.ev_pub.record(self.sL)
            L.iter_timer.lap()
            L.current_iter += self.K
        self.iterations += 1
        return stats

    def drain(self):
        self.torch.cuda.synchronize()


class SurrealDefaultLauncher(Launcher):
    def __init__(self, agent_class, learner_class, replay_class, session_config, env_config, learner_config,
                 eval_mode='eval_stochastic', agent_batch_size=8, eval_batch_size=8, render=False):
        self.agent_class = agent_class
        self.learner_class = learner_class
        self.replay_class = replay_class
        self.session_config = session_config
        self.env_config = env_config
        self.learner_config = learner_config
        self.eval_mode = eval_mode
        self.render = render
        self.agent_batch_size = agent_batch_size
        self.eval_batch_size = eval_batch_size
        self.log = U.get_logger('launcher')
        self.replay = self.learner = self.agent = None
        self.iterations = None               # engine steps `launch` runs (None: until interrupted)
        self.rollout_steps = self.updates_per_chunk = None     # ReplayEngine chunk shape (None: its defaults)

    # -- constructors the reference exposes (launcher.py:192-217, 317-332, 369-381) ----------------------
    def setup_replay(self, replay_id=0):
        self.replay = self.replay_class(self.learner_config, self.env_config, self.session_config, index=replay_id)
        return self.replay

    def setup_learner(self):
        self.learner = self.learner_class(learner_config=self.learner_config, env_config=self.env_config,
                                          session_config=self.session_config)
        if self.replay is not None:
            self.learner.attach_replay(self.replay)
        return self.learner

    def setup_agent(self, agent_id):
        np.random.seed(int(__import__('time').time() * 100000 % 100000))       # launcher.py:201
        self.agent = self.agent_class(learner_config=self.learner_config, env_config=self.env_config,
                                      session_config=self.session_config, agent_id=agent_id, agent_mode='training')
        return self.agent

    def setup_eval(self, eval_id):
        return self.agent_class(learner_config=self.learner_config, env_config=self.env_config,
                                session_config=self.session_config, agent_id=eval_id, agent_mode=self.eval_mode,
                                render=self.render)

    # -- engine -------------------------------------------------------------------------------------------
    def setup_engine(self, env=None):
        """replay -> learner -> agent, then the initial publish + fetch (learner/base.py:356-362,
        agent/base.py:234-242)."""
        if self.replay is None:
            self.setup_replay(0)
        if self.learner is None:
            self.setup_learner()
        if self.agent is None:
            self.setup_agent(0)
        self.learner.main_setup()
        self.agent.main_setup(env)
        return self.agent, self.replay, self.learner

    def run_engine(self, iterations=None, rollout_steps=None, pipelined=None, updates_per_chunk=None):
        """Run actors + learner.  A learner with ``learn_from_replay`` on a replay with ``sample_device`` (DDPG on the
        uniform replay) runs in a ReplayEngine: ``iterations`` counts its steps, ``updates_per_chunk`` defaults to one
        update per env step of the chunk.  pipelined (default when one rollout chunk yields exactly one learner batch):
        PipelinedEngine -- actors and learner on two concurrent streams.  Otherwise alternate a rollout chunk with
        as many learner iterations as the replay can feed."""
        agent, replay, learner = self.setup_engine()
        if hasattr(learner, 'learn_from_replay') and hasattr(replay, 'sample_device'):
            T = rollout_steps or self.rollout_steps or REPLAY_ROLLOUT_STEPS
            eng = ReplayEngine(agent, replay, learner, T, updates_per_chunk or self.updates_per_chunk or T)
            eng.prime()
            while iterations is None or eng.iterations < iterations:
                eng.step()
            eng.drain()
            return learner
        T = rollout_steps or self.learner_config.algo.stride
        n, stride = self.learner_config.algo.n_step, self.learner_config.algo.stride
        one_batch_per_chunk = (n == stride == T and agent.num_envs == self.learner_config.replay.batch_size and
                               hasattr(learner, 'replay_out_buffers'))
        if pipelined is None:
            pipelined = one_batch_per_chunk
        if pipelined:
            eng = PipelinedEngine(agent, replay, learner, T)
            eng.prime()
            while iterations is None or eng.iterations < iterations:
                eng.step()
            eng.drain()
            return learner
        it = 0
        while iterations is None or it < iterations:
            agent.main_loop(max_steps=T)
            while replay.start_sample_condition():
                learner.main_loop()
                it += 1
                if iterations is not None and it >= iterations:
                    break
        return learner

    def launch(self, component_name_in):
        name = component_name_in.split('-')[0] if '-' in component_name_in else component_name_in
        if name in ('learner', 'engine', 'all'):
            return self.run_engine(self.iterations)
        if name in ('agent', 'agents', 'eval', 'evals', 'replay', 'replay_worker') or name in _NOOP_COMPONENTS:
            self.log.warning('component "%s" is collapsed into the learner process of surreal_b200 '
                             '(one process per GPU); launch `learner` instead', component_name_in)
            return None
        raise ValueError('Unexpected component {}'.format(component_name_in))

    def run_learner(self, iterations=None):
        return self.run_engine(iterations)

    def run_agent(self, agent_id):
        return self.launch('agent-%s' % agent_id)

    def run_replay_worker(self, replay_id):
        return self.setup_replay(replay_id)
