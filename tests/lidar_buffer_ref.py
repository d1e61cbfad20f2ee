"""A literal restatement of the reference's LiDAR buffer: Accumulator::BUFFER_L (include/Headers/Accumulator.hpp:3) with

- push: Accumulator::receive_lidar -> add -> Buffer::push (src/Modules/Accumulator.cpp:39-48, src/Objects/Buffer.cpp:26-28), every
  point of a processed message push_front-ed in message order, so content[0] is the newest point INSERTED and across messages the
  order is arrival order, not time order;
- get: Accumulator::get (Accumulator.hpp:61-74) with Algorithms::binary_search (include/Headers/Utils.hpp:9-23);
- clear: Buffer::clear(TimeType) (Buffer.cpp:66-70).

Nothing is fixed.  Of m points whose time equals t2 exactly only min(m, 2) are returned, and on unsorted content the result
depends on the binary search's exact probe sequence.  This is the oracle of the device buffer (lv_lidar_*), of its host build
(tests/cpu_shim/lidar_ring.cpp) and of the windowed tick tests.  Points are (time, x, y, z) tuples; x, y, z are float32 values.
"""
import collections

import numpy as np


def binary_search(content, t, desc=True):
    """Algorithms::binary_search, line for line (`int` arithmetic: (low + high) / 2 of non-negatives truncates like //)"""
    low = 0
    high = len(content) - 1
    sign = 1.0 if desc else -1.0
    probes = []
    while high >= low:
        mid = (low + high) // 2
        probes.append(mid)
        if sign * content[mid][0] < sign * t:
            high = mid - 1
        else:
            low = mid + 1
    high -= 1
    if high < 0:
        return 0, probes
    return high, probes


class LidarBuffer:
    """Buffer<Point> as the Accumulator uses it for LiDAR points"""

    def __init__(self):
        self.content = collections.deque()

    def push_message(self, xyz, time):
        """`for (Point p : points) this->add(p);` -> Buffer::push -> content.push_front(p)"""
        xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
        time = np.asarray(time, np.float64)
        for (x, y, z), t in zip(xyz.tolist(), time.tolist()):
            self.content.appendleft((t, x, y, z))

    def get(self, t1, t2):
        """Accumulator::get(BUFFER_L, t1, t2): (xyz float32 (m, 3), time float64 (m,)), oldest inserted first"""
        c = self.content
        k_t2 = max(0, binary_search(c, t2, True)[0])
        result = collections.deque()
        for k in range(k_t2, len(c)):
            cnt = c[k]
            if t1 > cnt[0]:
                break
            if t2 >= cnt[0]:
                result.appendleft(cnt)
        return as_arrays(result)

    def clear(self, t):
        """Buffer::clear(t): pop_back while t >= back().time"""
        c = self.content
        while len(c) > 0 and t >= c[-1][0]:
            c.pop()

    def size(self):
        return len(self.content)

    def times(self):
        """content's times, content[0] first"""
        return np.array([p[0] for p in self.content], np.float64)


def as_arrays(points):
    pts = list(points)
    xyz = np.array([p[1:] for p in pts], np.float32).reshape(-1, 3)
    time = np.array([p[0] for p in pts], np.float64)
    return xyz, time
