"""TEST INFRASTRUCTURE -- numpy restatement of the counter-based random streams of the synthetic benchmark env and
of the batched PPOAgent.act sampling, so that tests can replay the exact N(0,1) draws of a device rollout.

Philox4x32-10 follows the published round function (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy
as 1, 2, 3", SC'11); the key schedule and the (counter, key) conventions are those of
surreal_b200/csrc/common.cuh / rollout.cu.  The synthetic env itself is SURVEY.md §8(d) cfg 2 (it has no
counterpart in the reference: the reference's envs are gym / MuJoCo adapters, out of scope):

    s' = tanh(Ws s + Wa a) + 0.01 xi,  r = -|s|^2 / D + 0.1 xi',  done when the episode reaches its cap.
"""
import numpy as np

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(seed, ctr_lo, ctr_hi):
    """Vectorised: seed / ctr_lo / ctr_hi broadcastable uint64 arrays -> four uint32 arrays."""
    seed = np.asarray(seed, dtype=np.uint64)
    ctr_lo = np.asarray(ctr_lo, dtype=np.uint64)
    ctr_hi = np.asarray(ctr_hi, dtype=np.uint64)
    seed, ctr_lo, ctr_hi = np.broadcast_arrays(seed, ctr_lo, ctr_hi)
    k0, k1 = seed & _M32, seed >> np.uint64(32)
    c0, c1 = ctr_lo & _M32, ctr_lo >> np.uint64(32)
    c2, c3 = ctr_hi & _M32, ctr_hi >> np.uint64(32)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    w0, w1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2                       # 32x32 -> 64-bit products (no overflow in uint64)
        hi0, lo0 = p0 >> np.uint64(32), p0 & _M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
    return c0.astype(np.uint32), c1.astype(np.uint32), c2.astype(np.uint32), c3.astype(np.uint32)


def box_muller(a, b):
    """Two N(0,1) from two 32-bit words (common.cuh: box_muller).  The uniforms and the angle are formed in fp32
    exactly as on the device; log / sqrt / cos / sin are then evaluated in float64, i.e. this returns the value the
    device's fp32 libm calls approximate to a few ulp."""
    f = np.float32
    u1 = (a.astype(np.float32) + f(1.0)) * f(2.3283064365386963e-10)
    u2 = b.astype(np.float32) * f(2.3283064365386963e-10)
    ang = (f(6.283185307179586) * u2).astype(np.float64)
    rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    return (rad * np.cos(ang)).astype(np.float32), (rad * np.sin(ang)).astype(np.float32)


def agent_eps(agent_seed, step, actor_ids, A):
    """N(0,1) draws of PPOAgent.act at global step `step` for actors `actor_ids` -> [len(ids), A] float32
    (common.cuh: action_noise4 -- key = agent seed, counter = (step, actor << 16 | j // 4))."""
    ids = np.asarray(actor_ids, dtype=np.uint64)[:, None]
    grp = np.arange((A + 3) // 4, dtype=np.uint64)[None, :]
    x, y, z, w = philox4x32_10(np.uint64(agent_seed), np.uint64(step), (ids << np.uint64(16)) | grp)
    a0, a1 = box_muller(x, y)
    b0, b1 = box_muller(z, w)
    out = np.stack([a0, a1, b0, b1], axis=-1).reshape(len(ids), -1)
    return out[:, :A]


def env_noise(env_seed, step, actor_ids, D):
    """(xi [n, D] on the successor state, xi' [n] on the reward, reset state [n, D]) of SyntheticEnv at `step`."""
    ids = np.asarray(actor_ids, dtype=np.uint64)[:, None]
    d = np.arange(D, dtype=np.uint64)[None, :]
    key = np.uint64(env_seed) ^ np.uint64(0x5851F42D4C957F2D)
    x, y, z, w = philox4x32_10(key, np.uint64(step), (ids << np.uint64(20)) | d)
    gx, gy = box_muller(x, y)
    rz, _ = box_muller(z, w)
    return gx, gy[:, 0], rz


def synth_env_step(state, action, Ws, Wa, env_seed, step, actor_ids):
    """One step of the synthetic env for the given actors: -> (obs_next fp32 [n, D], reward fp32 [n])."""
    f = np.float32
    D = state.shape[1]
    gx, gy, _ = env_noise(env_seed, step, actor_ids, D)
    acc = state.astype(np.float64) @ Ws.T.astype(np.float64) + action.astype(np.float64) @ Wa.T.astype(np.float64)
    nxt = np.tanh(acc).astype(np.float32) + f(0.01) * gx
    rew = (-(state.astype(np.float64) ** 2).sum(1) / D).astype(np.float32) + f(0.1) * gy
    return nxt.astype(np.float32), rew.astype(np.float32)
