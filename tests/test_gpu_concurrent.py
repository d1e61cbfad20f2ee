"""Several sequences on one GPU at once.  Handles share nothing, so a sequence must give the same bits whatever runs beside it:
every case below holds each sequence, tick by tick, to the same sequence run alone on a fresh handle (status, every iteration log,
x, P, last_time_updated, the map's points and the deferred errors).  The solo runs are themselves held to the references:
test_gpu_async_tick ties the windowed tick to the synchronous chain and the stages to the oracle, and the bench-shaped case here
checks one solo update evaluation by evaluation against the oracle (check_every_evaluation).

Cases: K handles on K streams enqueued round-robin from one thread; the same handles on one shared stream (graphs, direct
launches, direct launches without programmatic dependent launch: a kernel's stream predecessor then belongs to another handle);
one thread per sequence with a late create, a growing map and an early destroy beside the others; a caller stream created
without cudaStreamNonBlocking whose first update graph is captured while another thread creates a handle, and a capture on
such a stream held open for the whole of another thread's create; and bench.py's multi-sequence step at test size for
S = 1, 2, 4, 8.

Beside them, a CPU rule: no function of the library calls a legacy-stream or device-wide operation (synchronous cudaMemset /
cudaMemcpy*, cudaDeviceSynchronize).  On the legacy stream such a call waits for every blocking stream of the device, and while
another thread captures a graph on a blocking stream it breaks that capture or fails itself (cudaErrorStreamCaptureImplicit)."""
import ctypes as C
import glob
import os
import re
import threading
import time

import numpy as np
import pytest

from conftest import Scene, oracle_params
from test_device_buffers import _functions, _strip
from test_gpu_async_tick import Chain, make_path, same_result, tick_messages
from test_gpu_fullsize import check_every_evaluation

gpu = pytest.mark.gpu

N_TICKS = 12
SWITCHES = ("LV_NO_REUSE", "LV_NO_GRAPH", "LV_NO_PDL", "LV_SEARCH_GROUP")


def tick_time(i):
    return 10.1 + 0.1 * i


class Sequence:
    def __init__(self, name, sc, msgs, path, x2):
        self.name, self.sc, self.msgs, self.path, self.x2 = name, sc, msgs, path, x2


class Runner(Chain):
    """a Chain whose messages are all in device memory before its first tick, so that a tick only enqueues work: no message
    upload, which would synchronise the handle's stream between two handles' ticks"""

    def __init__(self, lv, seq, stream=None, max_map_points=1 << 18, **kw):
        super().__init__(lv, seq.sc, seq.msgs, seq.path, seq.x2, stream=stream, max_map_points=max_map_points, **kw)
        self.seq = seq
        self.d_msgs = [self.b.upload(g["raw"]) for g in seq.msgs]

    def tick(self, i):
        self.d_msg = self.d_msgs[i]
        self.enqueue(self.msgs[i], tick_time(i))

    def snapshot(self):
        """everything a caller reads back after a tick; synchronises the handle's stream"""
        return self.result(), self.loc.map_points(), self.loc.async_status()


def same_snapshot(got, ref, what):
    same_result(got[0], ref[0], what)
    assert got[1].shape == ref[1].shape, (what, got[1].shape, ref[1].shape)
    assert (got[1].view(np.uint32) == ref[1].view(np.uint32)).all(), what
    assert got[2] == ref[2], (what, got[2], ref[2])


def solo_run(lv, seq, **kw):
    """the sequence alone on a fresh handle (its own stream), a snapshot after every tick"""
    r = Runner(lv, seq, **kw)
    out = []
    for i in range(N_TICKS):
        r.tick(i)
        out.append(r.snapshot())
    info = r.loc.map_info()
    r.close()
    return out, info


@pytest.fixture(scope="module")
def sequences(lv, O, scene_xaloc, scene_kitti, scene_ouster, tmp_path_factory):
    scenes = [("xaloc", scene_xaloc), ("kitti", scene_kitti), ("ouster", scene_ouster),
              ("xaloc-2", Scene(lv, O, "xaloc.yaml", seed=20260931, max_map_points=1 << 19, max_points=1 << 16))]
    out = []
    for k, (name, sc) in enumerate(scenes):
        msgs = tick_messages(lv, sc, tmp_path_factory.mktemp(name), n_ticks=N_TICKS)
        path, x2 = make_path(lv, sc, seed=9 + k)
        out.append(Sequence(name, sc, msgs, path, x2))
    return out


@pytest.fixture(scope="module")
def solo(lv, sequences):
    """per sequence: the snapshots of its solo run, which must be real work (updates that ran, a map that grew), so that the
    comparisons below are not between empty results"""
    out = []
    for seq in sequences:
        snaps, _ = solo_run(lv, seq)
        statuses = [s[0][0] for s in snaps]
        assert statuses.count(lv.OK) >= N_TICKS // 2, (seq.name, statuses)
        assert len(snaps[-1][1]) > 1000 and all(s[2] == (lv.OK, "") for s in snaps), seq.name
        out.append(snaps)
    return out


# ---- one thread, K handles ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fetch", ["every_round", "at_end"])
def test_own_streams_round_robin_equal_the_solo_runs(lv, sequences, solo, fetch):
    """K handles on K streams; each round enqueues one tick of every handle, with no host wait between the handles"""
    import torch
    streams = [torch.cuda.Stream() for _ in sequences]
    runs = [Runner(lv, seq, stream=st.cuda_stream) for seq, st in zip(sequences, streams)]
    for i in range(N_TICKS):
        for r in runs:
            r.tick(i)
        if fetch == "every_round":
            for k, r in enumerate(runs):
                same_snapshot(r.snapshot(), solo[k][i], (r.seq.name, i))
    for k, r in enumerate(runs):
        same_snapshot(r.snapshot(), solo[k][-1], (r.seq.name, "end"))
        r.close()


@gpu
@pytest.mark.parametrize("switches", [(), ("LV_NO_GRAPH",), ("LV_NO_GRAPH", "LV_NO_PDL")],
                         ids=["graphs", "direct", "direct-no-pdl"])
def test_one_shared_stream_interleaved_equal_the_solo_runs(lv, sequences, solo, monkeypatch, switches):
    """the K handles on one caller stream, their ticks interleaved.  With direct launches (LV_NO_GRAPH, read by lv_create) the
    first kernel of a handle's update follows another handle's last kernel in the stream, so with programmatic dependent launch
    its prologue overlaps a kernel of another handle"""
    import torch
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k in switches:
        monkeypatch.setenv(k, "1")
    stream = torch.cuda.Stream()
    runs = [Runner(lv, seq, stream=stream.cuda_stream) for seq in sequences]
    for i in range(N_TICKS):
        for r in runs:
            r.tick(i)
        for k, r in enumerate(runs):
            same_snapshot(r.snapshot(), solo[k][i], (r.seq.name, switches, i))
    for r in runs:
        r.close()


# ---- one thread per sequence -------------------------------------------------------------------------------------------------
class Worker(threading.Thread):
    """runs one sequence on its own stream; records its snapshots, or the exception that ended it"""

    def __init__(self, lv, seq, stream, ticks=N_TICKS, start_after=None, done_with=None, **kw):
        super().__init__(daemon=True)
        self.lv, self.seq, self.stream, self.ticks, self.kw = lv, seq, stream, ticks, kw
        self.start_after, self.done_with = start_after, done_with
        self.snaps, self.error, self.info = [], None, None

    def run(self):
        r = None
        try:
            if self.start_after is not None:
                assert self.start_after.wait(300)
            r = Runner(self.lv, self.seq, stream=self.stream, **self.kw)
            for i in range(self.ticks):
                r.tick(i)
                self.snaps.append(r.snapshot())
                if self.done_with is not None and i == 2:
                    self.done_with.set()
            self.info = r.loc.map_info()
        except BaseException as e:                                # reported by the test's thread
            self.error = e
        finally:
            if self.done_with is not None:
                self.done_with.set()
            if r is not None:
                r.close()


def join_all(workers):
    for w in workers:
        w.join(600)
    assert not any(w.is_alive() for w in workers)
    for w in workers:
        assert w.error is None, (w.seq.name, repr(w.error))


@gpu
def test_threads_with_a_late_create_a_growing_map_and_an_early_destroy_equal_the_solo_runs(lv, sequences, solo):
    """K Python threads, one sequence each on its own stream (ctypes lets go of the GIL inside the library): the second creates
    its handle only once the first has ticked three times, the third starts from a 4096-point map that grows, the fourth destroys
    its handle half-way while the others tick"""
    import torch
    grow = dict(growth=1 << 20, max_map_points=4096)
    grow_solo, grow_info = solo_run(lv, sequences[2], **grow)
    assert grow_info["growths"] > 0, grow_info
    streams = [torch.cuda.Stream() for _ in sequences]
    third_tick = threading.Event()
    half = N_TICKS // 2
    workers = [Worker(lv, sequences[0], streams[0].cuda_stream, done_with=third_tick),
               Worker(lv, sequences[1], streams[1].cuda_stream, start_after=third_tick),
               Worker(lv, sequences[2], streams[2].cuda_stream, **grow),
               Worker(lv, sequences[3], streams[3].cuda_stream, ticks=half)]
    for w in workers:
        w.start()
    join_all(workers)
    refs = [solo[0], solo[1], grow_solo, solo[3][:half]]
    for w, ref in zip(workers, refs):
        assert len(w.snaps) == len(ref), w.seq.name
        for i, (got, want) in enumerate(zip(w.snaps, ref)):
            same_snapshot(got, want, (w.seq.name, i))
    assert workers[2].info["growths"] == grow_info["growths"], (workers[2].info, grow_info)


CAPTURE_THREAD_LOCAL = 1                                          # cudaStreamCaptureModeThreadLocal


def cudart():
    """the CUDA runtime the library links (libcudart.so.12, already loaded by the library: dlopen returns that copy)"""
    rt = C.CDLL("libcudart.so.12")
    rt.cudaStreamCreateWithFlags.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
    rt.cudaStreamDestroy.argtypes = [C.c_void_p]
    rt.cudaStreamBeginCapture.argtypes = [C.c_void_p, C.c_int]
    rt.cudaStreamEndCapture.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    rt.cudaGraphDestroy.argtypes = [C.c_void_p]
    return rt


@gpu
def test_blocking_caller_stream_captures_beside_a_create_in_another_thread(lv, sequences, solo):
    """A sequence on a caller stream created without cudaStreamNonBlocking, which synchronises with the legacy default stream.
    While its handle captures its first update graph (the first tick whose update runs), another thread creates a handle: a
    clear or copy of lv_create on the legacy stream at that moment would be an implicit dependency on a capturing stream, which
    CUDA rejects.  Both must succeed, and the sequence must keep its solo bits; the new handle then runs its own sequence."""
    lv.lib()
    rt = cudart()
    s = C.c_void_p()
    assert rt.cudaStreamCreateWithFlags(C.byref(s), 0) == 0
    seq, other = sequences[0], sequences[1]
    go = threading.Barrier(2)
    created, spans = {}, {}

    def create():
        go.wait(60)
        t0 = time.perf_counter()
        try:
            created["runner"] = Runner(lv, other)                 # lv_create, then the runner's buffers and messages
        except Exception as e:
            created["error"] = e
        spans["create"] = (t0, time.perf_counter())

    r = Runner(lv, seq, stream=s.value)
    got, t = [], None
    try:
        # tick 0 finds the map empty on the host and enqueues no update; tick 1 is the first to enqueue one, so its
        # correct_device_async captures the update graph of its sweep size
        r.tick(0)
        got.append(r.snapshot())
        t = threading.Thread(target=create, daemon=True)
        t.start()
        go.wait(60)
        t0 = time.perf_counter()
        r.tick(1)
        spans["capture tick"] = (t0, time.perf_counter())
        t.join(300)
        assert not t.is_alive()
        print("blocking stream, from the barrier: %s" % {k: "%.2f..%.2f ms" % (1e3 * (a - t0), 1e3 * (b - t0)) for k, (a, b) in spans.items()})
        assert "error" not in created, repr(created["error"])
        got.append(r.snapshot())
        for i in range(2, N_TICKS):
            r.tick(i)
            got.append(r.snapshot())
        for i, (a, b) in enumerate(zip(got, solo[0])):
            same_snapshot(a, b, (seq.name, "blocking stream", i))
    except BaseException:
        if "runner" in created:
            created["runner"].close()
        raise
    finally:
        if t is not None:
            t.join(300)
        r.close()
        assert rt.cudaStreamDestroy(s) == 0
    run_to_the_solo_bits(created["runner"], solo[1], "created beside the capture")


def run_to_the_solo_bits(r, ref, what):
    for i in range(N_TICKS):
        r.tick(i)
        same_snapshot(r.snapshot(), ref[i], (r.seq.name, what, i))
    r.close()


@gpu
def test_a_create_while_a_blocking_stream_is_being_captured(lv, sequences, solo):
    """The same hazard held open for the whole create: this thread begins a capture on a blocking stream, in the thread-local mode
    the library captures its update graphs in, and ends it only after another thread's handle is created and its messages are on
    the device.  Nothing of that may join the capture (CUDA would fail the call and invalidate the capture): the create must
    succeed, the capture must end without an error, and the new handle must run its sequence to its solo bits."""
    lv.lib()
    rt = cudart()
    s, graph, created = C.c_void_p(), C.c_void_p(), {}
    assert rt.cudaStreamCreateWithFlags(C.byref(s), 0) == 0

    def create():
        try:
            created["runner"] = Runner(lv, sequences[1])
        except Exception as e:
            created["error"] = e

    try:
        assert rt.cudaStreamBeginCapture(s, CAPTURE_THREAD_LOCAL) == 0
        t = threading.Thread(target=create, daemon=True)
        t.start()
        t.join(300)
        ended = rt.cudaStreamEndCapture(s, C.byref(graph))
        rt.cudaGetLastError()                                     # a failed capture's error must not reach the next CUDA call
        assert not t.is_alive()
        assert (ended, repr(created.get("error"))) == (0, "None"), (ended, created)
        assert rt.cudaGraphDestroy(graph) == 0
    except BaseException:
        if "runner" in created:
            created["runner"].close()
        raise
    finally:
        assert rt.cudaStreamDestroy(s) == 0
    run_to_the_solo_bits(created["runner"], solo[1], "created during a capture")


# ---- bench.py's multi-sequence step at test size -----------------------------------------------------------------------------
BENCH_RINGS, BENCH_AZIMUTHS, BENCH_MAP, BENCH_SWEEPS, BENCH_STEPS = 32, 512, 100_000, 4, 4


@pytest.fixture(scope="module")
def bench_sequences(lv, O):
    """bench.make_scene's sequences at test size: 16 384-point sweeps against 100 000-point maps, eight seeds"""
    n = BENCH_RINGS * BENCH_AZIMUTHS
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=BENCH_MAP + 4 * n, max_points=n)
    out = []
    for s in range(8):
        world = lv.SynthWorld(20261000 + 10 * s, BENCH_MAP)
        rng = np.random.default_rng(700 + s)
        sweeps, x_props = [], []
        for i in range(BENCH_SWEEPS):
            truth = world.pose(15.0 + 1.5 * i, prm)
            sweeps.append(world.sweep(truth, rings=BENCH_RINGS, azimuths=BENCH_AZIMUTHS, min_dist=4.0, range_sigma=0.02, seed=100 + i))
            d = np.zeros(23)
            d[0:3] = rng.uniform(-0.05, 0.05, 3)
            d[3:6] = rng.uniform(-0.5, 0.5, 3) * np.pi / 180.0
            x_props.append(O.boxplus(truth, d))
        out.append(dict(map=world.map(), sweeps=sweeps, x_props=x_props))
    x0, P0 = lv.init_state_host(prm)
    return dict(prm=prm, n=n, seqs=out, P0=P0)


def bench_leg(lv, torch, B, first, S):
    """multi_sequence_leg's step for sequences first .. first + S - 1: set_state on every handle, an L2 flush and a fork event on
    stream 0, one correct_device per stream, the join on stream 0; then every handle's logs and state"""
    streams = [torch.cuda.Stream() for _ in range(S)]
    flush = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    locs, sweeps = [], []
    for s in range(S):
        prm = lv.Params.from_buffer_copy(B["prm"])
        prm.stream = streams[s].cuda_stream
        loc = lv.Localizer(prm)
        loc.map_build(B["seqs"][first + s]["map"])
        locs.append(loc)
        sweeps.append([loc.upload(sw) for sw in B["seqs"][first + s]["sweeps"]])
    out = [[] for _ in range(S)]
    for i in range(BENCH_STEPS):
        for s in range(S):
            locs[s].set_state(B["seqs"][first + s]["x_props"][i % BENCH_SWEEPS], B["P0"])
        with torch.cuda.stream(streams[0]):
            flush.fill_(i & 255)
        fork, join = torch.cuda.Event(), torch.cuda.Event()
        fork.record(streams[0])
        ends = []
        for s in range(S):
            if s:
                streams[s].wait_event(fork)
            locs[s].correct_device(sweeps[s][i % BENCH_SWEEPS], B["n"])
            e = torch.cuda.Event()
            e.record(streams[s])
            ends.append(e)
        for e in ends[1:]:
            streams[0].wait_event(e)
        join.record(streams[0])
        for s in range(S):
            st, logs = locs[s].last_logs()
            x, P = locs[s].get_state()
            out[s].append((st, logs, x, P))
    join.synchronize()
    return locs, sweeps, out


def close_leg(locs, sweeps):
    for loc, ds in zip(locs, sweeps):
        for d in ds:
            loc.device_free(d)
        loc.close()


@gpu
def test_bench_multi_sequence_step_equals_one_sequence(lv, O, bench_sequences):
    """every sequence of S = 2, 4, 8 concurrent ones gives its S = 1 bits in every step (logs, x, P); the first sequence's
    first S = 1 update is held to the oracle evaluation by evaluation"""
    import torch
    B = bench_sequences
    alone = []
    for s in range(8):
        locs, sweeps, out = bench_leg(lv, torch, B, s, 1)
        alone.append(out[0])
        assert all(st == lv.OK and len(logs) >= 2 and logs[0]["n_matches"] > 5000 for st, logs, x, P in out[0]), s
        if s == 0:
            om = O.Map(O.KNN_REF_IKDTREE if O.ref_available() else O.KNN_KDTREE)
            om.build(B["seqs"][0]["map"])
            st, logs, x, P = out[0][0]
            check_every_evaluation(O, om, oracle_params(O, B["prm"]), B["seqs"][0]["x_props"][0], B["P0"], B["seqs"][0]["sweeps"][0],
                                   logs, locs[0], P_gpu=P)
        close_leg(locs, sweeps)
    for S in (2, 4, 8):
        locs, sweeps, out = bench_leg(lv, torch, B, 0, S)
        for s in range(S):
            for i, ((st, logs, x, P), (st1, logs1, x1, P1)) in enumerate(zip(out[s], alone[s])):
                same_result((st, logs, x, P, 0.0), (st1, logs1, x1, P1, 0.0), (S, s, i))
        close_leg(locs, sweeps)
    torch.cuda.empty_cache()


# ---- the sources: no legacy-stream or device-wide operation ------------------------------------------------------------------
PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "limo-velo_b200")
# the synchronous memsets and copies of the runtime (cudaMemset, cudaMemset2D, cudaMemcpy, cudaMemcpyToSymbol,
# cudaMemcpyFromSymbol, ...: every form without Async) and the device-wide waits
LEGACY = re.compile(r"\b(cuda(?:Memset|Memcpy)\w*?(?<!Async)|cudaDeviceSynchronize|cudaThreadSynchronize)\s*\(")
# (function, call): why it may stay
ALLOWED_LEGACY = {
    ("lv_debug_step_clocks", "cudaMemcpyFromSymbol"): "tuning build only (LV_STEP_TIMING): reads the step kernel's device-global clocks",
    ("lv_debug_probes", "cudaDeviceSynchronize"): "tuning build only (LV_STEP_TIMING): the probe counters are device-global",
    ("lv_debug_probes", "cudaMemcpyFromSymbol"): "tuning build only (LV_STEP_TIMING): reads the device-global probe counters",
    ("lv_debug_probes", "cudaMemcpyToSymbol"): "tuning build only (LV_STEP_TIMING): resets the device-global probe counters",
    ("lv_debug_timeline", "cudaDeviceSynchronize"): "tuning build only (LV_STEP_TIMING): the timeline table is device-global",
    ("lv_debug_timeline", "cudaMemcpyFromSymbol"): "tuning build only (LV_STEP_TIMING): reads the device-global timeline table",
    ("lv_debug_timeline", "cudaMemcpyToSymbol"): "tuning build only (LV_STEP_TIMING): resets the device-global timeline table",
}


def test_no_legacy_stream_or_device_wide_operations():
    sources = sorted(glob.glob(os.path.join(PKG, "csrc", "*.cu")) + glob.glob(os.path.join(PKG, "host", "*.cpp")))
    assert len(sources) >= 15
    found, offenders, names = set(), [], set()
    for f in sources:
        code = _strip(open(f).read())
        calls = [m.group(1) for m in LEGACY.finditer(code)]
        in_functions = 0
        for name, body in _functions(code):
            names.add(name)
            for m in LEGACY.finditer(body):
                in_functions += 1
                found.add((name, m.group(1)))
                if (name, m.group(1)) not in ALLOWED_LEGACY:
                    offenders.append("%s: %s calls %s" % (os.path.basename(f), name, m.group(1)))
        assert in_functions == len(calls), "%s: a call outside every function" % f
    assert not offenders, "on the handle's stream instead (cudaMemsetAsync / cudaMemcpyAsync / cudaStreamSynchronize): " + "; ".join(
        sorted(set(offenders)))
    assert {"create_buffers", "init_pairs", "lv_create", "launch_measure"} <= names
    assert found == set(ALLOWED_LEGACY), sorted(set(ALLOWED_LEGACY) - found)
