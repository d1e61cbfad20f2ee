"""The front-end restatements (frontend_ref) against the oracle, on the edge-case families of frontend_cases.  CPU only.

The voxel grid and the temporal decimator are restated operation by operation in fp32, so they must equal the oracle bit for
bit.  Deskew is restated in 50 digits; the oracle (fp32, glibc sinf / cosf) must lie within K u32 M of it, M being the largest
magnitude in a point's chain, and on the inconsistent paths that bar also pins the segment the oracle picked."""
import numpy as np
import pytest

import frontend_cases as FC
import frontend_ref as F

VOXEL = {name: (xyz, leaf) for name, xyz, leaf in FC.voxel_cases()}
TEMPORAL = {c[0]: c[1:] for c in FC.temporal_cases()}


@pytest.fixture(scope="module")
def deskew(O):
    return {c["name"]: c for c in FC.deskew_cases(O)}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", [n for n in VOXEL if n != "wrap"])
def test_voxel_restatement_equals_oracle(O, name):
    xyz, leaf = VOXEL[name]
    r = F.voxelgrid(xyz, leaf)
    if r["overflow"]:
        with pytest.raises(ValueError):
            O.voxelgrid_downsample(xyz, leaf)
        return
    ref = O.voxelgrid_downsample(xyz, leaf)
    assert ref.shape == r["out"].shape and (bits(ref) == bits(r["out"])).all()
    assert r["count"].sum() == len(xyz)


def test_voxel_wrap_case_wraps():
    """In the wrap case div_b[0] * div_b[1] exceeds INT32_MAX while dx * dy * dz does not, so PCL's int index wraps.  The
    oracle computes it with the same int arithmetic, which is signed overflow (undefined behaviour in C++), so it is not a
    yardstick there: the kernel is compared with the restatement's explicit wrap (test_gpu_frontend.py)."""
    xyz, leaf = VOXEL["wrap"]
    r = F.voxelgrid(xyz, leaf)
    c = r["cells"]
    assert c["divb"][0] * c["divb"][1] > F.INT32_MAX and c["mul"][2] < 0
    ex = c["ijk"][:, 0] + c["ijk"][:, 1] * c["divb"][0] + c["ijk"][:, 2] * c["divb"][0] * c["divb"][1]
    assert (ex >= 2 ** 32).any() and r["count"].sum() == len(xyz)
    assert len(r["count"]) < len(np.unique(ex))


@pytest.mark.parametrize("name", list(VOXEL))
def test_voxel_restatement_is_a_mean(name):
    """the restatement's own sanity: every point in exactly one leaf, every centroid within count u32 max|p| of the exact mean"""
    xyz, leaf = VOXEL[name]
    r = F.voxelgrid(xyz, leaf, exact=True)
    if r["overflow"]:
        return
    assert r["count"].sum() == len(xyz) and (np.diff(r["key"].astype(np.int64)) > 0).all()
    tol = r["count"][:, None] * F.U32 * np.abs(xyz).max()
    assert (np.abs(r["out"].astype(np.float64) - r["mean"]) <= tol).all()


@pytest.mark.parametrize("name", list(TEMPORAL))
def test_temporal_restatement_equals_oracle(O, name):
    xyz, rate, md = TEMPORAL[name]
    assert (F.temporal(xyz, rate, md) == O.temporal_downsample(xyz, rate, md)).all()


@pytest.mark.parametrize("name", FC.DESKEW_NAMES)
def test_oracle_deskew_within_bar_of_50_digits(O, deskew, name):
    c = deskew[name]
    q, seg, M = F.compensate(c["path"], c["Xt2"], c["xyz"], c["t"])
    assert (seg == c["seg"]).all()
    qo = O.compensate(c["path"], c["Xt2"], c["xyz"], c["t"])
    assert qo.shape == c["xyz"].shape                           # the walk keeps every point
    e = np.abs(qo - q).max(axis=1)
    assert (e <= FC.K * F.U32 * M).all(), (e / (F.U32 * M)).max()
    if c["inconsistent"]:
        FC.deskew_separation(c, (q, seg, M))                    # so the oracle's segment is the walk's, point by point
