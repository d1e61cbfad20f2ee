"""A restatement of the time-ordered merge of a message into the LiDAR buffer (lv_lidar_merge_device_async), beside
lidar_buffer_ref (the reference's Buffer / Accumulator::get) and full_points_ref (the same buffer of whole Points).

Let L be the live content in ascending position (oldest inserted first; the deque's content reversed) and B the message.

- The split s is one past the highest position of L whose time is <= B[0].time (0 when there is none), found by walking down from
  the newest point.  T_tail = L[s:].
- The order rule: every element of T_tail and of B is in order with its successor (the last one with itself): neither time is NaN
  and the successor's is not smaller.
- Refusals, the buffer unchanged: the n points do not fit the capacity ("full"); in order, but T_tail holds more points than the
  merge reserve ("overlap").
- In order ("write"): L becomes L[:s] + std::merge(T_tail, B) by time, T_tail first on equal times.
- Not in order ("append"): B is pushed as Buffer::push does, and the caller is told.
- An empty B changes nothing.
- Each point of B is first moved by rt_apply(T, p) = RotTransl * Point (RotTransl.cpp:43-48) in fp32, each product and sum
  rounded in lv_point_math.h's order: (R[r0] x + R[r1] y) + R[r2] z, then + t[r].  No T: the points as they are.

The buffers here subclass lidar_buffer_ref.LidarBuffer and full_points_ref.LidarBufferFull, so get and clear are the reference's.
"""
import numpy as np

import full_points_ref as FP
import lidar_buffer_ref as R

f32 = np.float32


def rt_apply(T, xyz):
    """RotTransl * Point in fp32: T = 12 floats (R row-major, then t)"""
    T = np.asarray(T, f32).reshape(12)
    xyz = np.asarray(xyz, f32).reshape(-1, 3)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    out = np.empty_like(xyz)
    for r in range(3):
        out[:, r] = ((T[3 * r] * x + T[3 * r + 1] * y) + T[3 * r + 2] * z) + T[9 + r]
    assert out.dtype == f32
    return out


def in_order(a, b):
    return a == a and b == b and not b < a


def run_in_order(times):
    return all(in_order(times[i], times[min(i + 1, len(times) - 1)]) for i in range(len(times)))


def split_of(L, b0):
    """the walk: one past the highest position whose time is <= b0"""
    for p in range(len(L) - 1, -1, -1):
        if L[p][0] <= b0:
            return p + 1
    return 0


def std_merge(a, b):
    """std::merge(a, b) by time with operator<: b's element goes first only when strictly older"""
    out, i, j = [], 0, 0
    while i < len(a) or j < len(b):
        if i < len(a) and (j >= len(b) or not b[j][0] < a[i][0]):
            out.append(a[i])
            i += 1
        else:
            out.append(b[j])
            j += 1
    return out


def merge_into(content, B, cap, reserve):
    """the merge of the point tuples B (time first) into the deque `content` (newest first); returns the mode"""
    n = len(B)
    if n == 0:
        return "write"
    L = list(reversed(content))
    if len(L) + n > cap:
        return "full"
    s = split_of(L, B[0][0])
    tail = L[s:]
    if not (run_in_order([p[0] for p in tail]) and run_in_order([p[0] for p in B])):
        content.extendleft(B)
        return "append"
    if len(tail) > reserve:
        return "overlap"
    content.clear()
    content.extendleft(L[:s] + std_merge(tail, B))
    return "write"


def message(xyz, time, T, lanes=None):
    """the message as point tuples in the primary frame: (t, x, y, z) or (t, x, y, z, intensity, range)"""
    xyz = np.asarray(xyz, f32).reshape(-1, 3)
    if T is not None:
        xyz = rt_apply(T, xyz)
    time = np.asarray(time, np.float64)
    cols = [time.tolist()] + [xyz[:, c].tolist() for c in range(3)]
    if lanes is not None:
        cols += [np.asarray(v, f32).tolist() for v in lanes]
    return list(zip(*cols))


class MergeBuffer(R.LidarBuffer):
    """the plain buffer with the merge; cap and reserve as lv_lidar_reserve / lv_lidar_reserve_merge"""

    def __init__(self, cap=float("inf"), reserve=float("inf")):
        super().__init__()
        self.cap, self.reserve = cap, reserve

    def merge_message(self, xyz, time, T=None):
        return merge_into(self.content, message(xyz, time, T), self.cap, self.reserve)


class MergeBufferFull(FP.LidarBufferFull):
    """the buffer of whole Points with the merge; a message without lanes brings intensity 0 and range 0"""

    def __init__(self, cap=float("inf"), reserve=float("inf")):
        super().__init__()
        self.cap, self.reserve = cap, reserve

    def merge_message(self, xyz, time, T=None, intensity=None, rng=None):
        n = len(time)
        lanes = (np.zeros(n, f32) if intensity is None else intensity, np.zeros(n, f32) if rng is None else rng)
        return merge_into(self.content, message(xyz, time, T, lanes), self.cap, self.reserve)


def compose(T_a, T_b):
    """T_a * T_b (RotTransl * RotTransl) in float64, for building test extrinsics; returns 12 floats"""
    A, B = np.asarray(T_a, np.float64), np.asarray(T_b, np.float64)
    Ra, Rb = A[:9].reshape(3, 3), B[:9].reshape(3, 3)
    return np.concatenate([(Ra @ Rb).ravel(), Ra @ B[9:] + A[9:]])


def random_extrinsic(rng, angle=0.3, shift=0.5):
    """a rotation about a random axis and a translation, as 12 float32 values"""
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = rng.uniform(-angle, angle)
    K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    Rm = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    return np.concatenate([Rm.ravel(), rng.uniform(-shift, shift, 3)]).astype(f32)


def content_arrays(buf, columns):
    """content (newest first) as arrays: time, and the `columns` values after it (x, y, z[, intensity, range])"""
    pts = list(buf.content)
    t = np.array([p[0] for p in pts], np.float64)
    rest = np.array([p[1:] for p in pts], f32).reshape(len(pts), columns)
    return t, rest

