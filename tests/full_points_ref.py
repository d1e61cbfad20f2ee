"""A restatement of what the reference does to a point's attributes between the message and the publishers, beside
lidar_buffer_ref (the buffer's index arithmetic) and frontend_ref.voxelgrid (the xyz centroids):

- BUFFER_L holds whole Points (include/Headers/Accumulator.hpp:3,61-74): push and get carry intensity and range with xyz and
  time.  A point pushed without them (the device's plain push onto a ring with lanes) has intensity 0 and range 0.
- Compensator::voxelgrid_downsample (src/Modules/Compensator.cpp:148-163) on full_info::Points: Processor::fill -> toPCL sets x,
  y, z, timestamp, intensity and range (Point.cpp:113-122); pcl::VoxelGrid<full_info::Point> with downsample_all_data_ = true goes
  through CentroidPoint, whose accumulators for this point type are AccumulatorXYZ and AccumulatorIntensity (an fp32 running sum
  from +0 in the leaf's order, then sum / (float)n); nothing accumulates timestamp or range, so they stay value-initialised (0).
  Point(const full_info::Point&) (Point.cpp:21-25) then sets intensity = the average, range = this->norm() of the CENTROID
  (set_attributes runs after set_XYZ, Point.cpp:164-168) and time = p.timestamp = 0.  On a cell-index overflow PCL hands the
  input on unchanged, but Compensator.cpp:161 still builds every output point with Point(p): xyz, intensity and time are the
  input's, and range is this->norm() of each point, not the input's range.  So the input range is never read.  PCL is not
  built here: this reading of PCL 1.8 is unpinned, as frontend_ref's is.
- Processor::fill's header stamp (PointCloudProcessor.cpp:125-133): starting from 0, the max of Conversions::sec2Microsec(t) =
  std::round(t * 1e6) as uint64 (Utils.cpp:14-16) over the points.  A downsampled cloud's times are all 0, so its stamp is 0,
  unless the voxel grid passed its input through: then the times, and so the stamp, are the input's.

Points of the buffer are (time, x, y, z, intensity, range) tuples; x, y, z, intensity and range are float32 values.
"""
import collections
import math

import numpy as np

import frontend_ref as F
import lidar_buffer_ref as R

f32 = np.float32


class LidarBufferFull:
    """Buffer<Point> of whole Points, content[0] the newest inserted (lidar_buffer_ref.LidarBuffer with the attributes)"""

    def __init__(self):
        self.content = collections.deque()

    def push_message(self, xyz, time, intensity=None, rng=None):
        """`for (Point p : points) this->add(p);` -> content.push_front(p); no attributes: 0 and 0"""
        xyz = np.asarray(xyz, f32).reshape(-1, 3)
        time = np.asarray(time, np.float64)
        n = len(time)
        intensity = np.zeros(n, f32) if intensity is None else np.asarray(intensity, f32)
        rng = np.zeros(n, f32) if rng is None else np.asarray(rng, f32)
        for (x, y, z), t, i, r in zip(xyz.tolist(), time.tolist(), intensity.tolist(), rng.tolist()):
            self.content.appendleft((t, x, y, z, i, r))

    def get(self, t1, t2):
        """Accumulator::get(BUFFER_L, t1, t2): (xyz (m, 3), time, intensity, range), oldest inserted first"""
        c = self.content
        k_t2 = max(0, R.binary_search(c, t2, True)[0])
        result = collections.deque()
        for k in range(k_t2, len(c)):
            cnt = c[k]
            if t1 > cnt[0]:
                break
            if t2 >= cnt[0]:
                result.appendleft(cnt)
        return as_arrays(result)

    def clear(self, t):
        c = self.content
        while len(c) > 0 and t >= c[-1][0]:
            c.pop()

    def size(self):
        return len(self.content)

    def times(self):
        return np.array([p[0] for p in self.content], np.float64)


def as_arrays(points):
    pts = list(points)
    xyz = np.array([p[1:4] for p in pts], f32).reshape(-1, 3)
    time = np.array([p[0] for p in pts], np.float64)
    return xyz, time, np.array([p[4] for p in pts], f32), np.array([p[5] for p in pts], f32)


def norm32(xyz):
    """Point::norm in fp32, the decoder's |p| (lv_wire.h wire_norm): sqrt((x x + y y) + z z), each step rounded"""
    xyz = np.asarray(xyz, f32).reshape(-1, 3)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    out = np.sqrt((x * x + y * y) + z * z)
    assert out.dtype == f32
    return out


def voxelgrid_full(xyz, time, intensity, leaf):
    """pcl::VoxelGrid<full_info::Point> then Point(const full_info::Point&): (xyz, time, intensity, range) of the leaves, ascending
    cell index, input order inside a leaf (frontend_ref.voxelgrid's order); range is always the norm of the output xyz"""
    xyz = np.ascontiguousarray(xyz, f32).reshape(-1, 3)
    time, intensity = np.asarray(time, np.float64), np.asarray(intensity, f32)
    if len(xyz) == 0:
        return xyz.copy(), np.zeros(0), np.zeros(0, f32), np.zeros(0, f32)
    v = F.voxelgrid(xyz, leaf)
    if v["overflow"]:
        return xyz.copy(), time.copy(), intensity.copy(), norm32(xyz)     # Point(p) of each passed point: set_attributes
    lanes = np.repeat(intensity[v["order"]][:, None], 3, axis=1)           # AccumulatorIntensity: the same running sum per leaf
    sums = F._seq_sums(lanes, v["starts"], v["count"])[:, 0]
    mean = sums / v["count"].astype(f32)
    assert mean.dtype == f32
    out = v["out"]
    return out, np.zeros(len(out)), mean, norm32(out)


def sec2microsec(t):
    """Conversions::sec2Microsec: std::round(t * 1e6) (half away from zero) as uint64; finite t >= 0 only"""
    x = float(t) * 1e6
    assert math.isfinite(x) and x >= 0.0, t
    r = math.floor(x)
    return int(r) + (1 if x - r >= 0.5 else 0)                                # x - floor(x) is exact


def stamp_us(times):
    """Processor::fill: pcl.header.stamp = 0, then the max of sec2Microsec over the points"""
    s = 0
    for t in np.asarray(times, np.float64).tolist():
        s = max(s, sec2microsec(t))
    return s
