"""Experience windowing on the actor side (reference: surreal/env/exp_sender_wrapper.py).

Both models consume a flat stream of ``(step_id, reward, done)`` per episode and emit what the
reference's wrappers would ``send`` -- expressed over step ids so they can be compared with the
HBM staging kernels index-for-index."""
from collections import deque


def multistep_windows(ep_lens, n_step, stride, reward_fn=None):
    """exp_sender_wrapper.py:153-264.  Returns a list of (obs_step_ids[n], obs_next_id, done_flags[n]).
    The deque is cleared on reset (:204-207), so windows never span episodes and the tail of an
    episode that does not fill a window is discarded; after a send, ``stride`` items are popped (:222-226)."""
    out = []
    g = 0
    for L in ep_lens:
        last = deque()
        for t in range(L):
            done = (t + 1 >= L)
            last.append((g, done))
            g += 1
            if len(last) == n_step:
                out.append(([s for s, _ in last], g, [d for _, d in last]))
                for _ in range(stride):
                    if last:
                        last.popleft()
    return out


def ssar_nstep(ep_lens, n_step, gamma, reward_fn):
    """exp_sender_wrapper.py:72-112.  Emits (obs_id, obs_next_id, action_id, reward, done).
    Reward accumulation uses exponent ``n_step - i - 1`` for deque position i (:105) -- the true age
    only once the deque is full; reproduced as written."""
    out = []
    g = 0
    for L in ep_lens:
        last = deque()
        for t in range(L):
            obs_id = g
            g += 1
            reward = reward_fn(g)
            done = (t + 1 >= L)
            for i, e in enumerate(last):
                e[1] = g
                e[3] += pow(gamma, n_step - i - 1) * reward
                e[4] = done
            last.append([obs_id, g, obs_id, reward, done])
            if len(last) == n_step:
                e = last.popleft()
                out.append(tuple(e))
    return out


class SsarBatch:
    """N actors of exp_sender_wrapper.py:72-112, each with its own deque, stepped in (step, actor) order, sending into
    one ``replay.Uniform`` ring: the k-th record sent lands in slot k % capacity, later records overwrite earlier ones.

    Sums are written as the reference writes them, ``e += pow(gamma, n_step - i - 1) * r`` on Python floats: the
    product is rounded to float64, then the sum.  A record is (obs, obs_next, action, reward, done) with the reward
    still a Python float; the HBM ring holds it rounded to float32.  Observations and actions are opaque payloads."""

    def __init__(self, N, n_step, gamma, capacity):
        from .replay import Uniform
        self.N, self.n_step, self.gamma = N, n_step, float(gamma)
        self.ring = Uniform(capacity, 0)
        self.total_in = 0
        self.steps = 0
        self.obs = [None] * N
        self.last_n = [deque() for _ in range(N)]

    def reset(self, obs):
        """_reset of every actor: s_0 per actor, deques cleared (exp_sender_wrapper.py:95-98)."""
        for i in range(self.N):
            self.obs[i] = obs[i]
            self.last_n[i].clear()

    def step(self, action, obs_next, reward, done, obs_reset=None):
        """_step of every actor in actor order (exp_sender_wrapper.py:100-112).  An actor whose episode ended is reset
        right after its step, to ``obs_reset[i]`` (``obs_next[i]`` when None), as the reference's driver loop resets."""
        n = self.n_step
        for i in range(self.N):
            r, d = float(reward[i]), bool(done[i])
            last = self.last_n[i]
            for k, e in enumerate(last):
                e[1] = obs_next[i]
                e[3] += pow(self.gamma, n - k - 1) * r
                e[4] = d
            last.append([self.obs[i], obs_next[i], action[i], r, d])
            if len(last) == n:
                self.ring.insert(tuple(last.popleft()))
                self.total_in += 1
            self.obs[i] = obs_next[i]
            if d:
                self.obs[i] = obs_next[i] if obs_reset is None else obs_reset[i]
                last.clear()
        self.steps += 1

    def pending(self, i):
        """Actor i's deque, oldest first: [(obs, action, float64 sum)]."""
        return [(e[0], e[2], e[3]) for e in self.last_n[i]]

    def state(self):
        """(next_idx, size, capacity, total_in) of the ring, as UniformReplay.state holds them."""
        return self.ring.next_idx, len(self.ring.mem), self.ring.memory_size, self.total_in
