"""Tuning aid: wall-clock timeline (ns of %globaltimer) of the kernels of one graph-replayed update.
Library built with `make EXTRA=-DLV_STEP_TIMING`."""
import ctypes, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as G, bench
lv = G.load_package()
CFG = os.environ.get("LV_TIMELINE_CFG", "cfg1")             # any of bench.CONFIGS but cfg4
prm = bench.config_params(lv, CFG)
world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=2, prm=prm, cfg=CFG)
x0, P0 = lv.init_state_host(prm)
loc = lv.Localizer(prm); loc.map_build(mp)
d = [loc.upload(s) for s in sweeps]
buf = (ctypes.c_ulonglong * 320)()
names = {1: "reuse", 2: "search", 3: "upper", 4: "fit", 5: "step"}
for it in range(6):
    loc.set_state(x_props[it % 2], P0)
    if it % 2: loc.flush_l2()
    loc.synchronize()
    loc.L.lv_debug_timeline(buf)            # reset
    pr = (ctypes.c_ulonglong * 2)(); loc.L.lv_debug_probes(pr)
    loc.correct_device(d[it % 2], len(sweeps[it % 2]))
    loc.synchronize()
    loc.L.lv_debug_timeline(buf)
    loc.L.lv_debug_probes(pr); print("hash probes in this update:", pr[0])
    t = np.array(buf[:], dtype=np.float64).reshape(5, 8, 8)
    valid = t[0] < 1.8e19
    t0 = t[0][valid].min()
    print(f"--- update {it} ({'flushed L2' if it % 2 else 'warm'}): us since the first kernel was scheduled; sched / first..last block past the wait / end of thread 0 | of any warp")
    for e in range(4):
        row = []
        for k in (1, 2, 3, 4, 5):
            if t[0][e][k] < 1.8e19:
                row.append(f"{names[k]} {1e-3 * (t[0][e][k] - t0):6.1f}/{1e-3 * (t[1][e][k] - t0):6.1f}..{1e-3 * (t[3][e][k] - t0):6.1f}/{1e-3 * (t[2][e][k] - t0):6.1f}|{1e-3 * (t[4][e][k] - t0):6.1f}")
        print(f"  eval {e}: " + "  ".join(row) + f"   [searched again {int(t[2][e][7])}, ring search {int(t[2][e][6])}]")
