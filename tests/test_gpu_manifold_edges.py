"""The manifold algebra at its edges (tests/manifold_cases.py) on the device, against the 50-digit IKFoM restatement
(tests/ikfom_mp.py): the lv_manifold.h functions in a kernel (tests/gpu_shim), lv_ieskf_step_kernel on every step family,
lv_predict_kernel from every heading, a 20 000-sample spinning run through lv_propagate_device, and rot_to_quat's second branch
through lv_init_state.  test_manifold_edges_ref.py runs the same families through the host build and the oracle."""
import numpy as np
import pytest

import filter_cases as FC
import gpu_shim_binding as GS
import ikfom_mp as M
import manifold_cases as MC
from test_manifold_edges_ref import _noise, _step_rows, check_init_state, check_long_run, rot_to_quat_matrices

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


@pytest.fixture(scope="module")
def bases(O, scene_xaloc, scene_kitti):
    return [FC.base(O, scene_xaloc), FC.base(O, scene_kitti)]          # kitti: estimate_extrinsics off, Q singular


def test_primitives_against_mp(O, bases):
    """every lv_manifold.h function compiled for the device within its bar of the 50-digit reference (manifold_cases.bar, the
    host build's bars), each row on the branch its label names; a non-finite output fails"""
    states = [c["x_prop"] for b in bases for c in MC.headings(O, b) + MC.charts(O, b)]
    rows = MC.primitive_rows(O, states)
    ops, inp = MC.pack(rows)
    worst = MC.primitive_errors(rows, GS.manifold(ops, inp))
    print("\n" + "\n".join("%-22s %.3f" % kv for kv in sorted(worst.items())))
    assert all(v <= 1.0 for v in worst.values()), worst


def test_step_edges(O, bases):
    """every step family of both scenes at the last evaluation (so the exit block runs): dx_, the iterate and P within
    8 kappa 2^-53 of the 50-digit evaluation, the degenerate and converged flags equal to its decisions; the table of errors
    is printed with -s"""
    def stepper(c, r, it, oprm):
        g = GS.step(c["x_prop"], c["P"], c["x_cur"], c["HTH"], c["HTh"], c["nm"], c["R"], c["D"], c["limits"], c["max_iter"],
                    c["est"], it=it, t=0, n_evals=c["max_iter"])
        assert g["status"] == 0 and g["done"] == 1
        assert g["degenerate"] == int(r["degenerate"]) and g["converged"] == int(r["conv"]), c["family"]
        e = MC.step_errors(c, r, g["dx"], g["x"])
        e["P"] = MC._err(g["P"], M.to_np(r["P"]))
        return e
    MC.print_step_table(_step_rows(O, bases, stepper), "device vs mp (dx, x, P)")


def test_predict_from_every_heading(O, bases):
    """one launch of the predict kernel from every heading of both scenes (both signs) over 6 samples with |omega| dt of 0.5,
    1.5 and 3 rad, and one sample on each side of so3_exp's Taylor bound, against the 50-digit esekf::predict"""
    for b in bases:
        sc = b["scene"]
        noise = _noise(sc.prm)
        for name, x in MC.heading_states(O, b):
            acc, gyr, dts = MC.imu_samples(len(name), x, 6, (0.5, 1.5, 3.0))
            xg, Pg = GS.predict(x, sc.P0, acc, gyr, dts, noise)
            xm, Pm = x, sc.P0
            for i in range(len(dts)):
                xm, Pm = M.predict(xm, Pm, acc[i], gyr[i], dts[i], *noise)
            xm, Pm = M.to_np(xm), M.to_np(Pm)
            assert np.abs(xg - xm).max() <= 64 * U * max(1.0, np.abs(xm).max()), name
            assert np.abs(Pg - Pm).max() <= 64 * U * np.abs(Pm).max(), name
    scene_xaloc = bases[0]["scene"]
    noise = _noise(scene_xaloc.prm)
    x = bases[0]["x_prop"].copy()
    for k in (-2, -1, 0, 1):
        w = MC.taylor_omega(k)
        assert ((2.0 ** -8) ** 2 * (w * w) < MC.TAYLOR) == (k < 0)
        xg, Pg = GS.predict(x, scene_xaloc.P0, [-x[23:26]], [[w, 0, 0]], [2.0 ** -7], noise)
        xm, Pm = M.predict(x, scene_xaloc.P0, -x[23:26], [w, 0, 0], 2.0 ** -7, *noise)
        assert np.abs(xg - M.to_np(xm)).max() <= 8 * U * np.abs(x).max(), k
        assert np.abs(Pg - M.to_np(Pm)).max() <= 64 * U * np.abs(M.to_np(Pm)).max(), k


def test_long_spinning_run(lv, O, scene_xaloc):
    """20 000 samples at 400 Hz spinning at 10 rad/s through lv_propagate_device: x against a 30-digit state-only
    propagation, P against np.longdouble, the quaternion's norm drift following the oracle's (neither renormalises)"""
    prm = scene_xaloc.prm
    x0 = scene_xaloc.x_prop.copy()
    acc, gyr, dts = MC.spin_run(x0)
    loc = lv.Localizer(prm)
    loc.set_state(x0, scene_xaloc.P0)
    loc.propagate_device(acc, gyr, dts)
    x, P = loc.get_state()
    loc.close()
    xo, Po = x0.copy(), scene_xaloc.P0.copy()
    for i in range(len(dts)):
        xo, Po = O.predict(xo, Po, acc[i], gyr[i], dts[i], *_noise(prm))
    check_long_run(x0, scene_xaloc.P0, acc, gyr, dts, _noise(prm), x, P, xo)


def test_rot_to_quat_through_init_state(lv, O):
    """lv_init_state on a handle: offset_R_L_I from I_Rotation_L with trace <= 0 (rot_to_quat's second branch) and > 0,
    against Eigen's Quaternion(Matrix3) in 50 digits and the oracle bit for bit"""
    def init(prm):
        loc = lv.Localizer(prm)
        loc.init_state()
        x, P = loc.get_state()
        loc.close()
        return x, P
    for R in rot_to_quat_matrices():
        check_init_state(lv, O, R, init)
