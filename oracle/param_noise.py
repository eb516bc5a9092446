"""TEST INFRASTRUCTURE -- restatement of surreal/agent/param_noise.py:9-74 as the DDPG agent drives it
(ddpg_agent.py:136-153,173-175) and of the flat per-actor image layout of the device implementation.

The reference perturbs a dict {module: {state_dict key: float32 array}} in float64 (``p + np.random.normal(0, sigma,
shape)``) and ``ModuleDict.load`` rounds the sum to float32 once (module_dict.py:47-63).  ``draw(shape)`` supplies the
N(0,1) draws (numpy's legacy ``normal(0, sigma)`` is ``0 + sigma * gauss``, so noise = sigma * z exactly).

AdaptiveNormalParameterNoise quirks kept as written: ``total_action_distance`` is OVERWRITTEN at every
``compute_dist_interval``-th act (not accumulated), so the mean is the latest distance over the number of acts since
the last apply; the distance and the mean are torch float32 scalars (also the comparison with the target), sigma is a
Python float (float64); the first apply adapts nothing when no act happened before it."""
import numpy as np
import torch

from .philox import philox4x32_10


def perturb(params, sigma, draw):
    """{key: float32} -> {key: float32 perturbed} (apply + ModuleDict.load), draws in key order."""
    out = {}
    for k, p in params.items():
        z = np.asarray(draw(p.shape), dtype=np.float64)
        out[k] = (p.astype(np.float64) + sigma * z).astype(np.float32)
    return out


class NormalParameterNoise:
    def __init__(self, sigma):
        self.sigma = float(sigma)

    def apply(self, params, draw):
        return perturb(params, self.sigma, draw)

    def compute_action_distance(self, original_action, modified_action):
        pass


class AdaptiveNormalParameterNoise:
    def __init__(self, target_stddev, compute_dist_interval=10, alpha=1.04, sigma=0.01):
        self.sigma = float(sigma)
        self.target_stddev = target_stddev
        self.compute_dist_interval = compute_dist_interval
        self.alpha = alpha
        self.i = 0
        self.total_action_distance = 0.0
        self.decisions = []              # 'up' / 'down' per adapting apply

    def compute_action_distance(self, original_action, modified_action):
        """actions: float32 [A] (the policy outputs before the action clip)."""
        if self.i % self.compute_dist_interval == 0:
            o, m = torch.as_tensor(original_action), torch.as_tensor(modified_action)
            self.total_action_distance = (((o - m) ** 2).sum()) ** 0.5
        self.i += 1

    def apply(self, params, draw):
        if self.i > 0:
            mean = self.total_action_distance / self.i
            if mean > self.target_stddev:
                self.sigma /= self.alpha
                self.decisions.append('down')
            else:
                self.sigma *= self.alpha
                self.decisions.append('up')
        self.i = 0
        return perturb(params, self.sigma, draw)


# -- flat per-actor images (surreal_b200/csrc/param_noise.cu) ------------------------------------------------------
def _ru(v, m):
    return (v + m - 1) // m * m


def flat_layout(dims):
    """[(w_off, b_off, K, N, ldw)] of the FlatNet kernel layout and the flat size."""
    lay, off = [], 0
    for l in range(len(dims) - 1):
        K, N = dims[l], dims[l + 1]
        ldw = _ru(N, 4)
        lay.append((off, off + K * ldw, K, N, ldw))
        off += K * ldw + ldw
    return lay, off


def image_stride(dims):
    """Floats per actor image: the flat size rounded up to 128 bytes."""
    return _ru(flat_layout(dims)[1], 32)


def to_flat(layers, dims, stride=None, dtype=np.float32):
    """[(weight [out, in], bias [out])] -> one flat image [stride] (W transposed to [in][ldw], padding zero)."""
    lay, size = flat_layout(dims)
    out = np.zeros(stride if stride is not None else size, dtype=dtype)
    for (w_off, b_off, K, N, ldw), (w, b) in zip(lay, layers):
        wt = np.zeros((K, ldw), dtype=dtype)
        wt[:, :N] = np.asarray(w).T
        out[w_off:w_off + K * ldw] = wt.reshape(-1)
        out[b_off:b_off + N] = np.asarray(b)
    return out


def from_flat(flat, dims):
    """Inverse of to_flat."""
    lay, _ = flat_layout(dims)
    layers = []
    for (w_off, b_off, K, N, ldw) in lay:
        w = np.asarray(flat[w_off:w_off + K * ldw]).reshape(K, ldw)[:, :N].T.copy()
        layers.append((w, np.asarray(flat[b_off:b_off + N]).copy()))
    return layers


def padding_mask(dims, stride):
    """bool [stride]: True at offsets that hold no parameter (ldw padding columns and the tail)."""
    ones = [(np.ones((dims[l + 1], dims[l])), np.ones(dims[l + 1])) for l in range(len(dims) - 1)]
    return to_flat(ones, dims, stride, dtype=np.float64) == 0.0


# -- the device's perturbation stream (surreal_b200/csrc/param_noise.cu) -----------------------------------------------
PARAM_NOISE_KEY = 0xC2B2AE3D27D4EB4F


def box_muller_f64(a, b):
    """Two float64 N(0,1) from two 32-bit words (param_noise.cu: box_muller_f64): uniforms and angle formed exactly
    as on the device, log / sqrt / cos / sin in float64 (the device's double libm agrees to an ulp or two)."""
    u1 = (a.astype(np.float64) + 1.0) * 2.3283064365386963e-10
    u2 = b.astype(np.float64) * 2.3283064365386963e-10
    ang = 6.283185307179586 * u2
    rad = np.sqrt(-2.0 * np.log(u1))
    return rad * np.cos(ang), rad * np.sin(ang)


def param_noise_unit(agent_seed, fetch, actor, stride):
    """float64 N(0,1) draws of the parameter-noise image of local actor `actor` at fetch `fetch` -> [stride], one per
    flat offset (padding offsets draw too and are discarded).  Philox4x32-10 (oracle/philox.py) with key = agent seed ^
    PARAM_NOISE_KEY and counter = (fetch, actor << 32 | offset // 4)."""
    grp = np.arange((stride + 3) // 4, dtype=np.uint64)
    key = np.uint64(agent_seed) ^ np.uint64(PARAM_NOISE_KEY)
    x, y, z, w = philox4x32_10(key, np.uint64(fetch), (np.uint64(actor) << np.uint64(32)) | grp)
    a0, a1 = box_muller_f64(x, y)
    b0, b1 = box_muller_f64(z, w)
    return np.stack([a0, a1, b0, b1], axis=-1).reshape(-1)[:stride]
