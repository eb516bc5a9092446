"""Float64 restatement of prioritized replay (surreal_b200.replay.PrioritizedReplay / csrc/replay_per.cu), after the
reference's prioritized_replay.py + segment_tree.py with its two bugs fixed (a record's own slot gets its priority; the
mass is drawn over the whole view, newest record included).

Trees in heap order over P = capacity rounded up to a power of two (>= 2): float32 leaves p^alpha (0: never inserted),
float64 internal sums (parent = left + right), min nodes where a 0 leaf counts as +inf.  ``PerRef`` adds admission at
max_priority^alpha, the view-restricted proportional descent for given u, the importance weights, the beta schedule and
the last-wins priority update."""
import numpy as np

from oracle.philox import philox4x32_10


def leaves_for(capacity):
    P = 2
    while P < capacity:
        P *= 2
    return P


def leaf_value(p, alpha):
    return np.float32(np.float64(np.float32(p)) ** np.float64(alpha))


class TreeRef:
    def __init__(self, capacity, leaf=None):
        self.cap = int(capacity)
        self.P = leaves_for(self.cap)
        self.leaf = np.zeros(self.P, np.float32) if leaf is None else np.array(leaf, np.float32).copy()
        self.sum = np.zeros(self.P, np.float64)
        self.mn = np.full(self.P, np.inf, np.float32)
        self.rebuild()

    def rebuild(self):
        P = self.P
        lv = self.leaf.astype(np.float64)
        lm = np.where(self.leaf > 0, self.leaf, np.float32(np.inf)).astype(np.float32)
        w = P // 2
        self.sum[w:P] = lv[0::2] + lv[1::2]
        self.mn[w:P] = np.minimum(lm[0::2], lm[1::2])
        while w > 1:
            h = w // 2
            self.sum[h:w] = self.sum[w:2 * w:2] + self.sum[w + 1:2 * w:2]
            self.mn[h:w] = np.minimum(self.mn[w:2 * w:2], self.mn[w + 1:2 * w:2])
            w = h

    def node_sum(self, i):
        return float(self.leaf[i - self.P]) if i >= self.P else float(self.sum[i])

    def node_min(self, i):
        if i >= self.P:
            v = self.leaf[i - self.P]
            return np.float32(v) if v > 0 else np.float32(np.inf)
        return self.mn[i]

    def range_sum(self, l, r):
        """sum of leaves [l, r), bottom-up, in the kernel's order"""
        left = right = 0.0
        l, r = l + self.P, r + self.P
        while l < r:
            if l & 1:
                left = left + self.node_sum(l)
                l += 1
            if r & 1:
                r -= 1
                right = self.node_sum(r) + right
            l, r = l >> 1, r >> 1
        return left + right

    def range_min(self, l, r):
        m = np.float32(np.inf)
        l, r = l + self.P, r + self.P
        while l < r:
            if l & 1:
                m = min(m, self.node_min(l))
                l += 1
            if r & 1:
                r -= 1
                m = min(m, self.node_min(r))
            l, r = l >> 1, r >> 1
        return np.float32(m)

    def descend(self, x):
        """find_prefixsum_idx (segment_tree.py:101-124)"""
        i = 1
        while i < self.P:
            left = self.node_sum(2 * i)
            if left > x:
                i = 2 * i
            else:
                x = x - left
                i = 2 * i + 1
        return i - self.P

    def view_sums(self, start, count):
        end = start + count
        end1, end2 = min(end, self.cap), max(0, end - self.cap)
        s1 = self.range_sum(start, end1)
        s = s1 + self.range_sum(0, end2) if end2 > 0 else s1
        m = self.range_min(start, end1)
        if end2 > 0:
            m = min(m, self.range_min(0, end2))
        return dict(base=self.range_sum(0, start), s1=s1, s=s, end1=end1, end2=end2, min=np.float32(m))

    def sample(self, start, count, us):
        """-> (slots, masses, S): the view-restricted descent for each u in [0, 1)"""
        v = self.view_sums(start, count)
        slots, masses = [], []
        for u in us:
            mass = float(u) * v['s']
            if v['end2'] == 0 or mass < v['s1']:
                x, lo, hi = v['base'] + mass, start, v['end1']
            else:
                x, lo, hi = mass - v['s1'], 0, v['end2']
            s = min(max(self.descend(x), lo), hi - 1)
            slots.append(s)
            masses.append(mass)
        return np.array(slots, np.int64), np.array(masses), v['s']

    def weights(self, slots, start, count, beta):
        """(leaf / min over the view)^(-beta) in float64"""
        m = float(self.view_sums(start, count)['min'])
        return (self.leaf[slots].astype(np.float64) / m) ** (-float(beta))

    def prefix_boundaries(self, start, count):
        """cumulative leaf sums over the view, in view order (for the near-boundary exception of a draw)"""
        order = [(start + r) % self.cap for r in range(count)]
        return np.cumsum(self.leaf[order].astype(np.float64))


def philox_u(seed, counter, batch):
    """u = (64-bit word >> 11) * 2^-53 of draw b: Philox call b // 2, words x:y (even b) or z:w (odd b)"""
    calls = np.arange((batch + 1) // 2, dtype=np.uint64)
    x, y, z, w = philox4x32_10(np.uint64(seed), np.uint64(counter), calls)
    us = []
    for b in range(batch):
        hi, lo = (x, y) if b % 2 == 0 else (z, w)
        word = (int(hi[b // 2]) << 32) | int(lo[b // 2])
        us.append((word >> 11) * 2.0 ** -53)
    return np.array(us)


def beta_schedule(t, beta0, anneal):
    """LinearSchedule(anneal, beta0 -> 1.0) of the reference DQN at step t; beta0 when anneal is None"""
    if anneal is None:
        return beta0
    return beta0 + min(float(t) / anneal, 1.0) * (1.0 - beta0)


class PerRef:
    def __init__(self, capacity, alpha):
        self.tree = TreeRef(capacity)
        self.alpha = float(alpha)
        self.max_priority = np.float32(1.0)
        self.admitted = 0

    def admit(self, total_in):
        cap = self.tree.cap
        gap = total_in - self.admitted
        slots = range(cap) if gap >= cap else [(self.admitted + k) % cap for k in range(gap)]
        v = leaf_value(self.max_priority, self.alpha)
        for s in slots:
            self.tree.leaf[s] = v
        self.admitted = total_in
        self.tree.rebuild()

    def update(self, indices, priorities):
        """prioritized_replay.py:137-143: sequential, so the last of equal indices wins"""
        for i, p in zip(np.asarray(indices).tolist(), np.asarray(priorities, np.float32).tolist()):
            self.tree.leaf[i] = leaf_value(p, self.alpha)
            self.max_priority = max(self.max_priority, np.float32(p))
        self.tree.rebuild()
