"""Results under concurrent use: one context from several caller streams, several contexts from one host thread, and contexts used
from several host threads at once (ctypes releases the GIL, so Python threads really run the library side by side).

Two pieces of state outlive a call and are shared between calls:
- the ring of K1 work counters of a context, one counter per staged launch, reused round-robin;
- the exposure times of the responseCalib streaming passes in constant memory, one copy per device, shared by every context.

Every result here is compared bit for bit with the same call run serially on one stream; the rest of the suite pins those serial
results to the oracle.  The serial run's outputs start as one sentinel and the concurrent run's as another, so a value that is
never written differs.  Where a test's point is an overlap, CUDA events show that the overlap happened, and the test fails and
says so if it did not.  Every test joins its threads and synchronises the device before it returns."""
import os
import threading
import time
import zipfile

import numpy as np
import pytest

from conftest import BIG_CALIBS, CALIBS
from mono_dataset_code_b200 import synthetic as S
from test_response_calib_scale import exposures, response_table, sweep_host

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

KINDS = ["uniform", "speckle", "gradient", "white", "black"] + ["uniform", "speckle", "gradient"] * 2
FLAGS = 15                       # rectify, gamma, vignette, NaN for overexposed pixels
FILL_SERIAL = {torch.float32: -12345.0, torch.float16: -1234.0, torch.uint8: 165, torch.float64: -7.0}
FILL_RUN = {torch.float32: -54321.0, torch.float16: -4321.0, torch.uint8: 90, torch.float64: -9.0}
_INT_VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mono_dataset_code_b200 import api as a
    return a


def mismatch(a, b, what):
    """None if a and b (CUDA or host tensors, numpy arrays) have the same shape, type and bits, else what differs."""
    a, b = (torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x for x in (a, b))
    if tuple(a.shape) != tuple(b.shape) or a.dtype != b.dtype:
        return f"{what}: {tuple(a.shape)} {a.dtype} against {tuple(b.shape)} {b.dtype}"
    ia, ib = (x.contiguous().view(_INT_VIEW[x.element_size()]) for x in (a, b))
    bad = (ia != ib).flatten()
    n = int(bad.sum())
    return f"{what}: {n} of {a.numel()} values differ from the serial run, the first at flat index {int(bad.nonzero()[0])}" if n else None


def assert_same(a, b, what):
    msg = mismatch(a, b, what)
    assert msg is None, msg


def timing_event():
    return torch.cuda.Event(enable_timing=True)


def run_threads(fns):
    """Run the callables on their own host threads, started together; re-raise the first exception once all have been joined."""
    gate = threading.Barrier(len(fns))
    results, errors = [None] * len(fns), []

    def body(i):
        try:
            gate.wait()
            results[i] = fns[i]()
        except BaseException as exc:         # raised again below, on the test's thread
            errors.append(exc)
        finally:
            torch.cuda.synchronize()

    threads = [threading.Thread(target=body, args=(i,)) for i in range(len(fns))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]
    return results


class Geometry:
    """One calibration: its models, the distinct frames on the device, and sentinel-filled output levels."""

    def __init__(self, api, root, cfg):
        self.iw, self.ih, self.ow, self.oh, mode, calib = cfg
        files = S.write_dataset_dir(root, self.iw, self.ih, self.ow, self.oh, mode, calib)
        self.u = api.UndistorterFOV(files["camera"])
        self.p = api.PhotometricUndistorter(files["pcalib"], files["vignette"], self.iw, self.ih)
        assert self.u.isValid() and self.p.validGamma and self.p.validVignette
        self.distinct = torch.from_numpy(np.stack([S.frame(i, self.iw, self.ih, k) for i, k in enumerate(KINDS)])).cuda()

    def context(self, api):
        return api.Context(self.u, self.p, 0)

    def batch(self, n, first=0):
        """n frames [n, ih*iw]; neighbours differ (position i holds distinct frame (7 (first + i) + 3) mod 11)."""
        idx = torch.tensor([(7 * (first + i) + 3) % len(KINDS) for i in range(n)], device="cuda")
        return self.distinct[idx].contiguous()

    def outputs(self, n, levels, fill, dtype=torch.float32):
        return [torch.full((n, (self.ow >> l) * (self.oh >> l)), fill[dtype], dtype=dtype, device="cuda") for l in range(levels)]


# -------------------------------------------------------------------------------------------------------- 1. K1's work counters
RING = 64                        # work counters per context (kCounterRing): every staged K1 launch takes the next one
N_LONG = 512                     # frames of the long call: milliseconds of work even with one CTA per SM
N_SHORT_CALLS = 140              # short calls: the ring wraps twice while the long call is in flight
SHORT_BATCHES = [(1, 0), (2, 1), (3, 3), (1, 6), (2, 7), (3, 9)]     # (frames, first): few distinct inputs, so TMA descriptors stay cached
LEVELS_K1 = 3                    # all three from the kernel's epilogue


@pytest.fixture(scope="module")
def c2(api, tmp_path_factory):
    return Geometry(api, str(tmp_path_factory.mktemp("c2")), BIG_CALIBS["c2_crop_1280"])


def sleep_cycles_per_ms():
    a, b = timing_event(), timing_event()
    a.record()
    torch.cuda._sleep(10_000_000)
    b.record()
    b.synchronize()
    return 10_000_000 / a.elapsed_time(b)


@pytest.mark.parametrize("order", ["long_first", "short_first"])
@pytest.mark.parametrize("loader", ["ldg", "tma", "hybrid"])
def test_work_counters_are_reused_in_order_across_streams(loader, order, api, c2):
    """One context, two caller streams, one CTA per SM so that both streams' kernels fit on the SMs side by side.  One stream runs
    one long call, the other 140 short calls, so the ring of 64 work counters wraps twice while the long call is in flight.

    long_first: the long call is issued first, and the 64th short call takes its counter.  short_first: the long call is issued
    after the short calls and takes the counter of the 77th.  Either way, the call that takes the counter second must wait until
    the other one has finished: zeroing a counter that a running launch draws from makes the two launches share item numbers,
    and tiles of one of them are never written.  To make the two calls meet, the long call and the second user of its counter
    (with the short calls behind it) wait for the end of a sleep on a third stream, which comes after every call has been issued:
    they are released at the same moment, and the short calls before the counter's second user have finished by then."""
    ctx = c2.context(api)
    if not ctx.loader_usable(loader):
        ctx.close()
        pytest.skip(f"the {loader} loader is not usable on this device")
    ctx.configure(loader, ctas_per_sm=1)
    long_in = c2.batch(N_LONG)
    short_in = [c2.batch(n, first) for n, first in SHORT_BATCHES]
    plan = [i % len(short_in) for i in range(N_SHORT_CALLS)]

    # serial: every distinct call once on one stream, with its launch count; then the short calls issued back to back, which
    # times their issue on the host and fills the descriptor caches
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        before = ctx.launch_count
        long_ref = c2.outputs(N_LONG, LEVELS_K1, FILL_SERIAL)
        ctx.prepare_batch(long_in, FLAGS, long_ref)
        s.synchronize()
        long_launches = ctx.launch_count - before
        short_ref, short_launches = [], []
        for x in short_in:
            before = ctx.launch_count
            short_ref.append(c2.outputs(x.shape[0], LEVELS_K1, FILL_SERIAL))
            ctx.prepare_batch(x, FLAGS, short_ref[-1])
            short_launches.append(ctx.launch_count - before)
        short_out = [c2.outputs(short_in[k].shape[0], LEVELS_K1, FILL_RUN) for k in plan]
        s.synchronize()
        t0 = time.perf_counter()
        for i, k in enumerate(plan):
            ctx.prepare_batch(short_in[k], FLAGS, short_out[i])
        issue_ms = (time.perf_counter() - t0) * 1e3
        s.synchronize()
    assert long_launches >= 1 and short_launches == [1] * len(short_in), (long_launches, short_launches)
    for outs in short_out:
        for o in outs:
            o.fill_(FILL_RUN[o.dtype])
    long_out = c2.outputs(N_LONG, LEVELS_K1, FILL_RUN)
    sleep_ms = 2.0 * issue_ms + 5.0
    sleep_cycles = int(sleep_cycles_per_ms() * sleep_ms)
    torch.cuda.synchronize()

    # `second`: the short call that takes the long call's counter (long_first), or whose counter the long call takes (short_first)
    second = RING - 1 if order == "long_first" else N_SHORT_CALLS - RING
    gate, sa, sb = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    start, released, long_done, first_short_done, before_second_done, second_done = (timing_event() for _ in range(6))
    with torch.cuda.stream(gate):
        start.record()
        torch.cuda._sleep(sleep_cycles)
        released.record()

    def issue_long():
        with torch.cuda.stream(sa):
            sa.wait_event(released)
            ctx.prepare_batch(long_in, FLAGS, long_out)
            long_done.record()

    def issue_short():
        with torch.cuda.stream(sb):
            for i, k in enumerate(plan):
                if i == second:
                    before_second_done.record()
                    sb.wait_event(released)
                ctx.prepare_batch(short_in[k], FLAGS, short_out[i])
                if i == 0:
                    first_short_done.record()
                if i == second:
                    second_done.record()

    before = ctx.launch_count
    for issue in ((issue_long, issue_short) if order == "long_first" else (issue_short, issue_long)):
        issue()
    gated = not released.query()
    torch.cuda.synchronize()
    at = {k: start.elapsed_time(e) - start.elapsed_time(released)
          for k, e in (("first", first_short_done), ("before", before_second_done), ("second", second_done), ("long", long_done))}
    timing = (f"after the release: short call 0 done at {at['first']:.2f} ms, short call {second - 1} at {at['before']:.2f} ms, "
              f"short call {second} at {at['second']:.2f} ms, the long call at {at['long']:.2f} ms")
    launches = ctx.launch_count - before
    bad = [mismatch(long_out[l], long_ref[l], f"{loader} {order}: long call, level {l}") for l in range(LEVELS_K1)]
    bad += [mismatch(short_out[i][l], short_ref[k][l], f"{loader} {order}: short call {i}, level {l}")
            for i, k in enumerate(plan) for l in range(LEVELS_K1)]
    bad = [m for m in bad if m]
    ctx.close()
    del long_in, long_ref, long_out, short_ref, short_out
    torch.cuda.empty_cache()                 # before any assertion: a failed test's frames would keep these gigabytes alive

    assert gated, f"the sleep of {sleep_ms:.1f} ms ended before every call was issued: the two calls were not released together"
    assert at["first"] < at["long"], f"the first short call finished after the long call: the streams did not overlap; {timing}"
    assert at["before"] <= 0, f"short call {second - 1} had not finished at the release; {timing}"
    assert launches == long_launches + sum(short_launches[k] for k in plan)
    assert not bad, f"{len(bad)} outputs differ from the serial run ({timing}): " + "; ".join(bad[:4])
    print(f"{loader} {order}: {timing}; {N_SHORT_CALLS} short calls issued in {issue_ms:.2f} ms")


# -------------------------------------------------------------------------------------------------------- 2-3. exposure times
RC_NPIX = 64 * 1024              # a multiple of 16 in a fresh (aligned) allocation: the streaming kernels, whose times sit in constant memory


def upload(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rc_problem(n, seed, npix=RC_NPIX):
    """data uint8 [n, npix], t [n], and a G and E to run the passes from, all on the device."""
    data, t = sweep_host(n, npix, seed)
    rng = np.random.default_rng(seed + 1)
    G = response_table() * rng.uniform(0.9, 1.1)
    E = rng.uniform(0.5, 40.0, npix)
    return dict(data=upload(data), t=upload(t), G=upload(G), E=upload(E))


def rc_pass(ctx, op, pr, fill):
    """One streaming pass into a new output buffer on torch's current stream: estep -> E [npix], rc_gstep -> G [256],
    rc_rmse_accumulate -> acc [2]."""
    npix = pr["data"].shape[1]
    if op == "estep":
        out = torch.full((npix,), fill, dtype=torch.float64, device="cuda")
        ctx.estep(pr["data"], pr["t"], pr["G"], out)
    elif op == "gstep":
        out = torch.full((256,), fill, dtype=torch.float64, device="cuda")
        ctx.rc_gstep(pr["data"], pr["t"], pr["E"], out)
    else:
        out = torch.zeros(2, dtype=torch.float64, device="cuda")
        ctx.rc_rmse_accumulate(pr["data"], pr["t"], pr["G"], pr["E"], out)
    return out


SLEEP_CYCLES = 20_000_000        # ~10 ms of spinning on a stream: the other stream's passes are issued and run meanwhile


def test_exposure_times_across_contexts_and_streams_on_one_thread(api):
    """Two contexts with their own streams on one host thread.  The E-step, the G-step and rmse alternate between the contexts, each
    with its own exposure times, and stream A's passes wait behind a sleep: the pass on stream B that refills the constant-memory
    times must wait for stream A's pass that still has to read them.  n = 1025 is one pass that reads the times from global
    memory, in the middle of the chain."""
    ctxs = [api.Context(None, None, 0), api.Context(None, None, 0)]
    chain = [(n, op) for n in (1, 8, 9, 1024) for op in ("estep", "gstep", "rmse")]
    chain.insert(len(chain) // 2, (1025, "estep"))
    problems = {(c, n): rc_problem(n, 100 * c + n) for c in (0, 1) for n in sorted({n for n, _ in chain})}
    serial = []
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for k, (n, op) in enumerate(chain):
            serial.append(rc_pass(ctxs[k % 2], op, problems[(k % 2, n)], FILL_SERIAL[torch.float64]))
            s.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    runs = []
    for k, (n, op) in enumerate(chain):
        with torch.cuda.stream(streams[k % 2]):
            if k % 2 == 0:
                torch.cuda._sleep(SLEEP_CYCLES)
            runs.append(rc_pass(ctxs[k % 2], op, problems[(k % 2, n)], FILL_RUN[torch.float64]))
    torch.cuda.synchronize()
    for k, (n, op) in enumerate(chain):
        assert_same(runs[k], serial[k], f"pass {k}: {op} n={n} on context {k % 2}")
    for c in ctxs:
        c.close()


N_ESTEP_PASSES = 200
ESTEP_N = 512


def test_exposure_times_across_host_threads_estep(api):
    """Two host threads, each with its own context and stream, run 200 E-steps each with their own exposure times per pass.  The
    constant-memory times are one copy per device: a pass may refill them only after every pass that read them before, whichever
    thread issued it."""
    rng = np.random.default_rng(7)
    probs = [rc_problem(ESTEP_N, 40 + th) for th in (0, 1)]
    times = [[upload(exposures(ESTEP_N, 1000 * th + k) * rng.uniform(0.5, 2.0)) for k in range(N_ESTEP_PASSES)] for th in (0, 1)]
    ctxs = [api.Context(None, None, 0), api.Context(None, None, 0)]

    def passes(th, fill):
        pr = probs[th]
        outs = [torch.full((RC_NPIX,), fill, dtype=torch.float64, device="cuda") for _ in range(N_ESTEP_PASSES)]
        for k in range(N_ESTEP_PASSES):
            ctxs[th].estep(pr["data"], times[th][k], pr["G"], outs[k])
        return outs

    serial = []
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for th in (0, 1):
            serial.append(passes(th, FILL_SERIAL[torch.float64]))
        s.synchronize()

    def thread(th):
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            outs = passes(th, FILL_RUN[torch.float64])
        st.synchronize()
        return outs

    runs = run_threads([lambda: thread(0), lambda: thread(1)])
    for th in (0, 1):
        for k in range(N_ESTEP_PASSES):
            assert_same(runs[th][k], serial[th][k], f"thread {th}, E-step {k}")
    for c in ctxs:
        c.close()


RC_LOOPS = 8


def test_exposure_times_across_host_threads_response_calib(api):
    """Two host threads, each with its own context, run the whole responseCalib loop (E-init, then four rounds of G-step, E-step,
    rescale and rmse after each) on different data at the same time, eight times over."""
    nits, n = 4, 200
    probs = [rc_problem(n, 60 + th) for th in (0, 1)]
    ctxs = [api.Context(None, None, 0), api.Context(None, None, 0)]

    def loop(th, fill):
        pr = probs[th]
        E = torch.full((RC_NPIX,), fill, dtype=torch.float64, device="cuda")
        G = torch.full((256,), fill, dtype=torch.float64, device="cuda")
        log = ctxs[th].response_calib(pr["data"], pr["t"], nits, E, G)
        return E, G, log

    serial = [loop(th, FILL_SERIAL[torch.float64]) for th in (0, 1)]
    runs = run_threads([lambda th=th: [loop(th, FILL_RUN[torch.float64]) for _ in range(RC_LOOPS)] for th in (0, 1)])
    for th in (0, 1):
        for r, run in enumerate(runs[th]):
            for what, a, b in zip(("E", "G", "log"), run, serial[th]):
                assert_same(a, b, f"thread {th}, loop {r}: {what}")
    for c in ctxs:
        c.close()


# -------------------------------------------------------------------------------------------------------- 4. isolation
SWEEP_FRAMES = 4
SWEEP_REPEATS = 3


@pytest.fixture(scope="module")
def c1(api, tmp_path_factory):
    return Geometry(api, str(tmp_path_factory.mktemp("c1")), CALIBS["c1_crop_640"])


def write_jpeg_sequence(api, folder, frames):
    """images.zip of the frames [n, h, w] (uint8 CUDA), encoded by the library's own JPEG encoder, and times.txt."""
    os.makedirs(folder, exist_ok=True)
    blobs = api.jpeg_encode_device(frames, 90)
    with zipfile.ZipFile(os.path.join(folder, "images.zip"), "w", zipfile.ZIP_STORED) as z:
        for i, b in enumerate(blobs):
            z.writestr(f"{i:05d}.jpg", b)
    with open(os.path.join(folder, "times.txt"), "w") as f:
        for i in range(len(blobs)):
            f.write(f"{i} {i * 0.05:.3f} 1.0\n")


class SweepInputs:
    """What one host thread's sweep reads: frames, a JPEG sequence, an irradiance and a small vignetteCalib problem, all its own."""

    def __init__(self, api, g, root, seed):
        self.g = g
        self.frames = g.batch(SWEEP_FRAMES, first=seed)
        self.frames_host = self.frames.cpu().numpy()
        write_jpeg_sequence(api, root, self.frames.view(SWEEP_FRAMES, g.ih, g.iw))
        self.seq_dir = root
        self.E = upload(np.random.default_rng(seed).uniform(0.0, 300.0, g.ow * g.oh))
        pr = S.vignette_calib_problem(5, 40, 30, 64, 48, seed=seed)
        self.vc = dict(images=upload(pr["images"]), p2x=upload(pr["p2x"]), p2y=upload(pr["p2y"]),
                       plane=pr["true_plane"], vig=pr["true_vignette"])


def sweep(api, ctx, inp, fill):
    """Every device entry point below once on `ctx`; those with a stream parameter run on torch's current stream.  Returns the
    results by name, on the host."""
    g, res = inp.g, {}
    for dtype in (torch.float32, torch.float16, torch.uint8):
        outs = g.outputs(SWEEP_FRAMES, 5, fill, dtype)
        ctx.prepare_batch(inp.frames, FLAGS, outs, dtype=dtype)
        for l, o in enumerate(outs):
            res[f"K1 {dtype} level {l}"] = o.cpu()
    host = [np.full((SWEEP_FRAMES, w * h), fill[torch.float32], np.float32) for w, h in ((g.ow >> l, g.oh >> l) for l in range(2))]
    ctx.prepare_batch_host(inp.frames_host, FLAGS, host)
    for l, o in enumerate(host):
        res[f"prepare_batch_host level {l}"] = o
    seq = api.Sequence(inp.seq_dir)
    assert seq.getNumImages() == SWEEP_FRAMES
    outs = g.outputs(SWEEP_FRAMES, 2, fill)
    seq.prepare_device(ctx, 0, SWEEP_FRAMES, True, True, True, True, levels=2, out=outs)
    torch.cuda.current_stream().synchronize()
    seq.close()
    for l, o in enumerate(outs):
        res[f"seq_prepare_device level {l}"] = o.cpu()
    blobs = api.jpeg_encode_device(inp.frames.view(SWEEP_FRAMES, g.ih, g.iw), 95, ctx=ctx)
    res["jpeg_encode_device"] = b"".join(len(b).to_bytes(8, "little") + b for b in blobs)
    dec = torch.full((SWEEP_FRAMES, g.ih, (g.iw + 15) // 16 * 16), fill[torch.uint8], dtype=torch.uint8, device="cuda")
    _, status = api.jpeg_decode_device(blobs, g.iw, g.ih, ctx=ctx, out=dec)
    res["jpeg_decode_device"], res["jpeg_decode_device status"] = dec.cpu(), status
    rect = torch.nan_to_num(res[f"K1 {torch.float32} level 0"].cuda(), nan=255.0).view(SWEEP_FRAMES, g.oh, g.ow)
    grey, mask = ctx.marker_threshold(rect)
    res["marker_threshold grey"], res["marker_threshold mask"] = grey.cpu(), mask.cpu()
    bgr, e16, rng = ctx.rc_plot_e(inp.E, g.ow, g.oh)
    res["rc_plot_e bgr"], res["rc_plot_e e16"], res["rc_plot_e range"] = bgr.cpu(), e16.cpu(), np.array(rng)
    vc = inp.vc
    plane = torch.from_numpy(vc["plane"].copy()).cuda()
    vig = torch.from_numpy(vc["vig"].copy()).cuda()
    st = ctx.vc_plane_step(vc["images"], vc["p2x"], vc["p2y"], 40, 30, 64, 48, vig, plane, 20.0 ** 2)
    st += ctx.vc_vignette_step(vc["images"], vc["p2x"], vc["p2y"], 40, 30, 64, 48, plane, vig, 20.0 ** 2)
    res["vc plane"], res["vc vignette"], res["vc stats"] = plane.cpu(), vig.cpu(), np.array(st)
    return res


def assert_same_results(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], bytes):
            assert a[k] == b[k], f"{what}: {k} differs from the serial run"
        else:
            assert_same(a[k], b[k], f"{what}: {k}")


def test_two_contexts_on_two_host_threads_are_isolated(api, c1, tmp_path):
    """Two host threads create their contexts at the same moment, then run the same sweep of device entry points, each on its own
    context, stream and data, three times over.  Each result must equal its serial run: state that two contexts share
    without ordering it shows up here as other bits."""
    inputs = [SweepInputs(api, c1, str(tmp_path / f"seq{th}"), 3 + 5 * th) for th in (0, 1)]
    torch.cuda.synchronize()
    ctxs = run_threads([lambda: c1.context(api), lambda: c1.context(api)])
    assert [c.auto_loader() for c in ctxs] == [ctxs[0].auto_loader()] * 2

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        serial = [sweep(api, ctxs[th], inputs[th], FILL_SERIAL) for th in (0, 1)]

    def thread(th):
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            return [sweep(api, ctxs[th], inputs[th], FILL_RUN) for _ in range(SWEEP_REPEATS)]

    runs = run_threads([lambda: thread(0), lambda: thread(1)])
    for th in (0, 1):
        for r, res in enumerate(runs[th]):
            assert_same_results(res, serial[th], f"thread {th}, round {r}")
    assert not any(np.array_equal(serial[0][k], serial[1][k]) for k in ("jpeg_decode_device", "vc plane")), "the threads' inputs must differ"
    for c in ctxs:
        c.close()
