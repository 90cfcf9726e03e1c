"""Stream ordering of every streaming entry point of ROMP and BEV (the two-slot pipeline), checked under injected delays.

Each model runs a batch's host-to-device copy on ``copy_stream``, its kernels on ``stream`` and its read-back on
``d2h_stream``; device inputs come from the caller's current stream and device results go back to it.  On an idle GPU a
missing wait between them rarely shows.  Here one stream at a time is held back by ~20 ms: every ``wait_event`` /
``wait_stream`` of a delayed stream is followed by ``torch.cuda._sleep`` on that stream (every internal stream starts its
work with such a wait), and a delayed caller sleeps on its own stream before it produces inputs and before it consumes
results.  A delay only changes which stream runs first, so a read that is not ordered after its producer sees stale
data on the first run: every scenario runs once and its results must equal, bit for bit, the synchronous path
(``forward_batch`` / ``forward_images`` / ``forward_video`` per batch) on a second instance with the same weights and
the same batch split.  The negative controls drop one wait each and require a mismatch, which shows the delays reach
the orderings the scenarios rely on."""
import contextlib
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

from oracle import preproc_oracle as P
from oracle import romp_oracle as O
from romp_b200 import ROMP, romp_settings, shard, synth
from romp_b200.bev import BEV, bev_settings
from romp_b200.staging import RawStager

pytestmark = pytest.mark.gpu

DELAY_MS = 20.0
MB = 3                                   # max_batch: lists and videos run in several chunks
DELAYS = ["copy", "kernel", "d2h", "caller"]
SIZES = [(480, 640), (640, 480), (300, 400), (512, 512), (720, 960), (37, 53), (1080, 1440)]


# ------------------------------------------------------------------------------------------------
# delay harness
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cycles():
    """torch.cuda._sleep cycles that take ~DELAY_MS at the clocks this GPU runs at now (measured with CUDA events)."""
    def timed(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        torch.cuda._sleep(n)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)
    timed(1000)
    probe = 1 << 22
    n = int(probe * DELAY_MS / timed(probe))
    ms = timed(n)
    print(f"\n[stream order] delay: {n} sleep cycles = {ms:.1f} ms (target {DELAY_MS:.0f} ms)")
    assert 0.5 * DELAY_MS < ms < 3 * DELAY_MS
    return n


class Harness:
    """Delays for one scenario.  ``delaying(streams, caller)`` patches torch.cuda.Stream.wait_event / wait_stream so that
    a stream among ``streams`` sleeps right after each of its waits; ``drop``: (stream, event) pairs whose wait is skipped."""

    def __init__(self, cycles):
        self.cycles = cycles
        self.delayed, self.caller, self.drop = set(), False, []

    def caller_sleep(self):
        """The caller's stream sleeps (when the scenario delays the caller)."""
        if self.caller:
            torch.cuda._sleep(self.cycles)

    @contextlib.contextmanager
    def delaying(self, streams=(), caller=False, drop=()):
        wait_event0, wait_stream0 = torch.cuda.Stream.wait_event, torch.cuda.Stream.wait_stream
        h = self

        def wait_event(s, event):
            if any(s.cuda_stream == st.cuda_stream and event is ev for st, ev in h.drop):
                return
            wait_event0(s, event)
            if s.cuda_stream in h.delayed:
                with torch.cuda.stream(s):
                    torch.cuda._sleep(h.cycles)

        def wait_stream(s, other):
            wait_event(s, other.record_event())

        self.delayed, self.caller, self.drop = {s.cuda_stream for s in streams}, caller, list(drop)
        torch.cuda.Stream.wait_event, torch.cuda.Stream.wait_stream = wait_event, wait_stream
        try:
            with torch.cuda.stream(torch.cuda.Stream()):         # the caller works on a stream of its own
                yield self
            torch.cuda.synchronize()
        finally:
            torch.cuda.Stream.wait_event, torch.cuda.Stream.wait_stream = wait_event0, wait_stream0
            self.delayed, self.caller, self.drop = set(), False, []


@pytest.fixture
def harness(cycles):
    return Harness(cycles)


def delayed_streams(m, which):
    return {"copy": [m.copy_stream], "kernel": [m.stream], "d2h": [m.d2h_stream], "caller": []}[which]


# ------------------------------------------------------------------------------------------------
# models, inputs, comparison
# ------------------------------------------------------------------------------------------------
def scenes(seed, n, sizes=SIZES):
    """n BGR images of mixed sizes: one smooth scene with per-image noise, so that no two images are alike."""
    rs = np.random.RandomState(seed)
    base = np.repeat(np.repeat(rs.randint(0, 256, (140, 190, 3)), 8, 0), 8, 1).astype(np.int32)
    out = []
    for i in range(n):
        h, w = sizes[(seed + i) % len(sizes)]
        tiled = np.tile(base, (-(-h // base.shape[0]), -(-w // base.shape[1]), 1))[:h, :w]
        img = np.clip(tiled + rs.randint(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)
        out.append(np.ascontiguousarray(img))
    return out


@pytest.fixture(scope="module")
def weights():
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    frames = np.concatenate([P.img_preprocess(x, 512)[0] for x in scenes(99, 4)])
    c, _ = O.romp_maps(sd, frames)
    sd, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    bev = synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)
    return dict(romp=(sd, pack), bev=bev)


@pytest.fixture(scope="module")
def models(weights):
    """get(kind, role, *flags): one instance per (kind, role, flags), its video state reset on every get.  role "ref"
    computes the references, role "run" the delayed scenarios."""
    cache = {}

    def get(kind, role, *flags):
        key = (kind, role, flags)
        if key not in cache:
            cache[key] = new(weights, kind, *flags)
        m = cache[key]
        if (m.temporal is not None) if kind == "romp" else m.temporal:
            m.reset_temporal()
        return m
    yield get
    cache.clear()


def new(weights, kind, *flags):
    if kind == "romp":
        return ROMP(romp_settings(list(flags)), state_dict=weights["romp"][0], smpl_pack=weights["romp"][1])
    w = weights["bev"]
    return BEV(bev_settings(list(flags)), state_dict=w[0], smpla_pack=w[1], smil_pack=w[2])


def flags(precision="bf16", *extra):
    return ("--precision", precision, "--max_batch", str(MB)) + tuple(extra)


def host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def snapshot(r):
    """A result (dict, None, or a list of them) as arrays of its own."""
    if isinstance(r, list):
        return [snapshot(x) for x in r]
    return None if r is None else {k: np.array(host(v)) for k, v in r.items()}


def diff(got, ref, where=""):
    """Every difference between two results (dicts / None / nested lists), as readable strings."""
    if isinstance(ref, list):
        if not isinstance(got, list) or len(got) != len(ref):
            return [f"{where}: {type(got).__name__} of {len(got) if isinstance(got, list) else '-'} vs list of {len(ref)}"]
        return [d for i, (g, r) in enumerate(zip(got, ref)) for d in diff(g, r, f"{where}[{i}]")]
    if (got is None) != (ref is None):
        return [f"{where}: {'None' if got is None else 'result'} vs {'None' if ref is None else 'result'}"]
    if ref is None:
        return []
    if set(got) != set(ref):
        return [f"{where}: keys {sorted(set(got) ^ set(ref))}"]
    out = []
    for k in ref:
        a, b = host(got[k]), host(ref[k])
        if a.dtype != b.dtype or a.shape != b.shape or not np.array_equal(a, b):
            out.append(f"{where}.{k}")
    return out


def persons(r):
    if isinstance(r, list):
        return sum(persons(x) for x in r)
    return 0 if r is None else len(r["cam"])


def fingerprint(r):
    """All cams of a result, flattened: neighbouring references must differ in them."""
    if isinstance(r, list):
        parts = [fingerprint(x) for x in r]
        return np.concatenate(parts) if parts else np.zeros(0)
    return np.zeros(0) if r is None else host(r["cam"]).astype(np.float64).ravel()


def check(got, ref, what):
    assert len(got) == len(ref), (what, len(got), len(ref))
    assert persons(ref) > 0, f"{what}: nobody detected, the scenario compares nothing"
    for a, b in zip(ref, ref[1:]):                  # a stale slot cannot match by accident
        fa, fb = fingerprint(a), fingerprint(b)
        assert fa.shape != fb.shape or not np.array_equal(fa, fb), f"{what}: neighbouring references are alike"
    bad = diff(got, ref)
    assert not bad, f"{what}: {len(bad)} mismatches, first {bad[:6]}"
    print(f"[stream order] {what}: {len(ref)} batches, {persons(ref)} persons bit-identical")


def pad_table():
    """Per-frame pad info [MB,6] on the device.  (Numpy offsets are copied from pageable memory, which blocks the host
    until the model's stream drains: a host sync in every batch that would hide a missing wait.)"""
    return torch.from_numpy(np.stack([P.img_preprocess(np.zeros(SIZES[k] + (3,), np.uint8), 512)[1]
                                      for k in range(MB)]).astype(np.float32)).cuda()


def romp_frames(n_batches, seed):
    """ROMP frame batches, their planted centre maps and one per-frame pad table (device)."""
    batches = [synth.synthetic_frames(MB, seed=seed + i) for i in range(n_batches)]
    planted, _ = synth.plant_centers(MB, seed=seed)
    return batches, planted, pad_table()


def bev_frames(n_batches, seed):
    batches = [synth.synthetic_frames(MB, seed=seed + i) for i in range(n_batches)]
    vol, _ = synth.plant_centers_3d(MB, seed=seed, kmax=6)
    return batches, vol, pad_table()


def bev_volume(n, seed):
    vol, _ = synth.plant_centers_3d(n, seed=seed, kmax=6)
    vol[1] = 0.0                                     # one image with nobody in it
    return vol


def frame_refs(m, kind, batches, override, offsets, **kw):
    """forward_batch per batch on the reference instance."""
    co = torch.from_numpy(override).cuda()
    if kind == "romp":
        return [snapshot(m.forward_batch(torch.from_numpy(b), offsets=offsets, center_override=co)) for b in batches]
    return [snapshot(m.forward_batch(torch.from_numpy(b), offsets=offsets, center3d_override=co, **kw)) for b in batches]


def stream_frames(m, kind, feed, override, offsets, to_numpy=True):
    kw = dict(center_override=override) if kind == "romp" else dict(center3d_override=override, img_max_side=640.0)
    return m.forward_batches(feed, offsets=offsets, to_numpy=to_numpy, **kw)


def consume_views(gen, h):
    """Consume a to_numpy=True stream: sleep on the caller's stream after each yield, and copy the arrays of batch i only
    once batch i+1 has been yielded and consumed, the end of their documented lifetime."""
    got, held = [], None
    for r in gen:
        h.caller_sleep()
        if held is not None:
            got.append(snapshot(held))
        held = r
    return got + [snapshot(held)]


# ------------------------------------------------------------------------------------------------
# 1. host frames refilled in one buffer (forward_batches), views held to the end of their lifetime
# ------------------------------------------------------------------------------------------------
HOST_CASES = [("romp", "bf16", "pinned"), ("romp", "bf16", "numpy"), ("bev", "bf16", "pinned"), ("bev", "bf16", "numpy"),
              ("romp", "fp32", "pinned"), ("bev", "fp32", "pinned")]


@pytest.mark.parametrize("delay", DELAYS)
@pytest.mark.parametrize("kind,precision,buf", HOST_CASES)
def test_host_frames_one_buffer(models, harness, kind, precision, buf, delay):
    batches, override, pads = (romp_frames if kind == "romp" else bev_frames)(4, 30)
    kw = {} if kind == "romp" else dict(img_max_side=640.0)
    ref = frame_refs(models(kind, "ref", *flags(precision)), kind, batches, override, pads, **kw)
    m = models(kind, "run", *flags(precision))
    one = torch.empty((MB, 512, 512, 3), dtype=torch.uint8).pin_memory() if buf == "pinned" else np.empty((MB, 512, 512, 3), np.uint8)

    def feed():
        for b in batches:
            h.caller_sleep()
            one[...] = torch.from_numpy(b) if buf == "pinned" else b      # refilled in place once the model has taken it
            yield one
    co = torch.from_numpy(override).cuda()
    with harness.delaying(delayed_streams(m, delay), delay == "caller") as h:
        got = consume_views(stream_frames(m, kind, feed(), co, pads), h)
    check(got, ref, f"{kind} {precision} forward_batches, one {buf} buffer, {delay} delayed")


# ------------------------------------------------------------------------------------------------
# 2. device inputs produced on a delayed caller stream, dropped right after submission
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("delay", DELAYS)
@pytest.mark.parametrize("kind", ["romp", "bev"])
def test_device_inputs_from_a_delayed_caller(models, harness, kind, delay):
    batches, override, pads = (romp_frames if kind == "romp" else bev_frames)(4, 40)
    kw = {} if kind == "romp" else dict(img_max_side=640.0)
    ref = frame_refs(models(kind, "ref", *flags()), kind, batches, override, pads, **kw)
    lists = [scenes(40 + j, n) for j, n in enumerate([3, 2, 5])]
    vol = bev_volume(5, 40)
    rm = models(kind, "ref", *flags())
    iref = [snapshot(rm.forward_images(li)) if kind == "romp" else
            snapshot(rm.forward_images(li, center3d_override=torch.from_numpy(vol[:len(li)]).cuda())) for li in lists]
    m = models(kind, "run", *flags())
    src = [torch.from_numpy(b).cuda() for b in batches]
    dev_lists = [[torch.from_numpy(x).cuda() for x in li] for li in lists]
    dev_override, dev_vol = (torch.from_numpy(x).cuda() for x in (override, vol))
    dev_pads = pads.clone()
    torch.cuda.synchronize()

    def produced(x):
        """A new tensor that the caller's stream writes x into after a sleep."""
        h.caller_sleep()
        return torch.empty(x.shape, dtype=x.dtype, device="cuda").copy_(x)

    def feed():
        for s in src:
            t = produced(s)
            yield t
            del t
            junk = torch.full(s.shape, 171, dtype=s.dtype, device="cuda")      # may take the memory of the frames just handed over
            del junk

    def image_feed():
        for li in dev_lists:
            imgs = []
            for k, x in enumerate(li):
                if k == 1:                               # a view with row stride > 3w
                    wide = torch.empty((x.shape[0], x.shape[1] + 7, 3), dtype=torch.uint8, device="cuda")
                    h.caller_sleep()
                    wide[:, :x.shape[1]] = x
                    imgs.append(wide[:, :x.shape[1]])
                    del wide
                else:
                    imgs.append(produced(x))
            yield imgs
            shapes = [t.shape for t in imgs]
            del imgs
            junk = [torch.full(s, 77, dtype=torch.uint8, device="cuda") for s in shapes]
            del junk

    streams = delayed_streams(m, delay)
    with harness.delaying(streams, caller=True) as h:
        co, offs = produced(dev_override), produced(dev_pads)
        gen = stream_frames(m, kind, feed(), co, offs)
        del co, offs
        got = consume_views(gen, h)
        vo = produced(dev_vol)
        igen = m.forward_image_batches(image_feed()) if kind == "romp" else m.forward_image_batches(image_feed(), center3d_override=vo)
        del vo
        igot = [snapshot(r) for r in igen]
    check(got, ref, f"{kind} forward_batches, device frames / overrides / offsets from the caller, {delay} delayed")
    check(igot, iref, f"{kind} forward_image_batches, device images from the caller, {delay} delayed")


# ------------------------------------------------------------------------------------------------
# 3. image lists: mixed sizes, several chunks per list, an empty list, staging buffers grown mid-stream
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("delay", DELAYS)
@pytest.mark.parametrize("kind", ["romp", "bev"])
def test_image_lists(models, harness, kind, delay):
    lists = [scenes(50, 7), [], scenes(51, 2), scenes(52, 4, sizes=[(300, 400), (640, 480), (480, 640)])]
    lists[3][2] = scenes(53, 1, sizes=[(2600, 2500)])[0]          # 19.5 MB: the slot's staging buffers grow mid-stream
    assert lists[3][2].nbytes > RawStager.MIN_BYTES > sum(x.nbytes for x in lists[0][:MB])
    vol = bev_volume(7, 50)
    co = torch.from_numpy(vol).cuda()
    kw = {} if kind == "romp" else dict(center3d_override=co)
    rm = models(kind, "ref", *flags())
    ref = [snapshot(rm.forward_images(li, **({} if kind == "romp" else dict(center3d_override=co[:len(li)])))) for li in lists]
    m = models(kind, "run", *flags())
    for slot in m.slots:                                           # fresh staging buffers, so that they grow here
        slot["raw"] = RawStager(m.tdevice)
    with harness.delaying(delayed_streams(m, delay), delay == "caller") as h:
        got = []
        for r in m.forward_image_batches(iter(lists), **kw):
            h.caller_sleep()
            got.append(snapshot(r))
    check(got, ref, f"{kind} forward_image_batches, {sum(map(len, lists))} images in {len(lists)} lists, {delay} delayed")


# ------------------------------------------------------------------------------------------------
# 4. video: tracker state and the reused pinned codes / signal slots across lists
# ------------------------------------------------------------------------------------------------
VIDEO_LISTS = [4, 2, 5, 3]


def video(seed):
    lists, k = [], 0
    frames = scenes(seed, sum(VIDEO_LISTS), sizes=[(480, 640), (512, 512), (640, 480)])
    for n in VIDEO_LISTS:
        lists.append(frames[k:k + n])
        k += n
    sids = [[(k // 3) % 2 for k in range(n)] for n in VIDEO_LISTS]
    return lists, sids


def walkers(T, seed, people=6):
    """3-D centre maps [T,64,128,128] of people walking through the volume."""
    rs = np.random.RandomState(seed)
    vol = rs.uniform(0, 0.05, size=(T, 64, 128, 128)).astype(np.float32)
    for _ in range(people):
        p, v, val = rs.uniform([24, 16, 16], [44, 112, 112]), rs.uniform(-1.5, 1.5, 3) * [0, 1, 1], rs.uniform(0.3, 0.9)
        for t in range(T):
            z, y, x = np.clip(np.round(p + v * t), [0, 2, 2], [63, 125, 125]).astype(int)
            vol[t, z, y, x] = max(vol[t, z, y, x], val)
    return vol


VIDEO_CASES = [("romp", ("-t",)), ("romp", ("-t", "--show_largest")), ("bev", ("-t",))]


def video_run(m, kind, lists, sids, vol, to_numpy=True):
    if kind == "romp":
        return m.forward_video_batches(iter(lists), iter(sids), to_numpy=to_numpy)
    return m.forward_image_batches(iter(lists), to_numpy=to_numpy, center3d_override=vol, signal_IDs=iter(sids))


def video_refs(m, kind, lists, sids, vol):
    if kind == "romp":
        return [snapshot(m.forward_video(li, s)) for li, s in zip(lists, sids)]
    return [snapshot(m.forward_images(li, center3d_override=vol[:len(li)], signal_IDs=s)) for li, s in zip(lists, sids)]


@pytest.mark.parametrize("delay", DELAYS)
@pytest.mark.parametrize("kind,mode", VIDEO_CASES)
def test_video(models, harness, kind, mode, delay):
    lists, sids = video(70)
    vol = torch.from_numpy(walkers(max(VIDEO_LISTS), 70)).cuda()
    ref = video_refs(models(kind, "ref", *flags("bf16", *mode)), kind, lists, sids, vol)
    m = models(kind, "run", *flags("bf16", *mode))
    with harness.delaying(delayed_streams(m, delay), delay == "caller") as h:
        got = []
        for r in video_run(m, kind, lists, sids, vol):
            h.caller_sleep()
            got.append(snapshot(r))
    check(got, ref, f"{kind} {' '.join(mode)} video in {len(lists)} lists, {delay} delayed")


# ------------------------------------------------------------------------------------------------
# 5. to_numpy=False: the consumer reads the device results on its own stream, late
# ------------------------------------------------------------------------------------------------
def own_copies(r):
    """Copies of a device result into buffers of the caller, enqueued on its current stream."""
    if isinstance(r, list):
        return [own_copies(x) for x in r]
    return None if r is None else {k: torch.empty_like(v).copy_(v) for k, v in r.items()}


def consume_device(gen, h):
    """After each yield the consumer sleeps on its stream, then copies every returned tensor into its own buffers, drops
    the result and pulls the next one; the copies are read only after the whole run."""
    kept = []
    for r in gen:
        torch.cuda._sleep(h.cycles)
        kept.append(own_copies(r))
        del r
    torch.cuda.current_stream().synchronize()
    return [snapshot(x) for x in kept]


DEVICE_CASES = ["romp batches", "bev batches", "romp images", "bev images", "romp video"]


@pytest.mark.parametrize("delay", DELAYS)
@pytest.mark.parametrize("case", DEVICE_CASES)
def test_device_results(models, harness, case, delay):
    kind, what = case.split()
    if what == "batches":
        batches, override, pads = (romp_frames if kind == "romp" else bev_frames)(4, 80)
        kw = {} if kind == "romp" else dict(img_max_side=640.0)
        ref = frame_refs(models(kind, "ref", *flags()), kind, batches, override, pads, **kw)
        m = models(kind, "run", *flags())
        co = torch.from_numpy(override).cuda()
        run = lambda: stream_frames(m, kind, (torch.from_numpy(b) for b in batches), co, pads, to_numpy=False)
    elif what == "images":
        lists = [scenes(81, 5), scenes(82, 2), [], scenes(83, 4)]
        vol = torch.from_numpy(bev_volume(5, 81)).cuda()
        kw = {} if kind == "romp" else dict(center3d_override=vol)
        ref = [snapshot(models(kind, "ref", *flags()).forward_images(li, **kw)) for li in lists]
        m = models(kind, "run", *flags())
        run = lambda: m.forward_image_batches(iter(lists), to_numpy=False, **kw)
    else:
        lists, sids = video(84)
        ref = video_refs(models(kind, "ref", *flags("bf16", "-t")), kind, lists, sids, None)
        m = models(kind, "run", *flags("bf16", "-t"))
        run = lambda: video_run(m, kind, lists, sids, None, to_numpy=False)
    with harness.delaying(delayed_streams(m, delay), delay == "caller") as h:
        got = consume_device(run(), h)
    check(got, ref, f"{case} to_numpy=False, read late on the caller's stream, {delay} delayed")


# ------------------------------------------------------------------------------------------------
# 6. the sharded path on one rank: the gather's pack reads a slot before its next batch overwrites it
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nccl_world1():
    mine = not dist.is_initialized()
    if mine:
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    yield
    if mine:
        dist.destroy_process_group()


@pytest.mark.parametrize("delay", ["gather", "copy", "kernel", "d2h"])
def test_sharded_gather_one_rank(models, harness, nccl_world1, delay):
    batches, override, pads = romp_frames(4, 90)
    ref = frame_refs(models("romp", "ref", *flags()), "romp", batches, override, pads)
    m = models("romp", "run", *flags())
    g = shard.ShardGather(1, m.record_layout(), capacity=m.cap)
    co = torch.from_numpy(override).cuda()
    feed = (torch.from_numpy(b).pin_memory() for b in batches)
    with harness.delaying([g.stream] if delay == "gather" else delayed_streams(m, delay)):
        got, gathered = [], []
        for own, handle in m.forward_batches(feed, offsets=pads, center_override=co, gather=g, frame_offset=0):
            got.append(snapshot(own))
            gathered.append(g.result(handle, to_numpy=True))
    check(got, ref, f"romp forward_batches(gather=) on one rank, {delay} delayed")
    for i, (a, b) in enumerate(zip(gathered, ref)):
        assert not diff(a, None if b is None else {k: b[k] for k in a}, f"gathered batch {i}")


# ------------------------------------------------------------------------------------------------
# 7. negative controls: without the one wait that orders a persistent buffer's reader after its writer, the delay
#    turns into a mismatch; with the wait restored the same run matches
# ------------------------------------------------------------------------------------------------
def control(h, m, run, ref, streams, drop, what):
    with h.delaying(streams, drop=drop):
        bad = diff(run(), ref)
    assert bad, f"{what}: dropping the wait changed nothing: the delay does not reach it"
    with h.delaying(streams):
        good = diff(run(), ref)
    assert not good, f"{what}: {good[:6]}"
    print(f"[stream order] control {what}: {len(bad)} mismatches without the wait, none with it")


def test_control_romp_kernels_wait_for_the_copy(weights, models, harness):
    """ROMP _submit_frames: stream waits for the slot's h2d event before its kernels read the frames."""
    batches, override, pads = romp_frames(4, 100)
    ref = frame_refs(models("romp", "ref", *flags()), "romp", batches, override, pads)
    m, co = new(weights, "romp", *flags()), torch.from_numpy(override).cuda()
    run = lambda: [snapshot(r) for r in m.forward_batches((torch.from_numpy(b).pin_memory() for b in batches), offsets=pads,
                                                          center_override=co)]
    control(harness, m, run, ref, [m.copy_stream], [(m.stream, s["h2d"]) for s in m.slots], "romp stream -> h2d, copy delayed")


def test_control_bev_preprocessing_waits_for_the_upload(weights, models, harness):
    """BEV _submit_images: stream waits for the slot's h2d event before the preprocessing reads the staged images."""
    lists = [scenes(101, 4), scenes(102, 3), scenes(103, 5)]
    vol = torch.from_numpy(bev_volume(5, 101)).cuda()
    ref = [snapshot(models("bev", "ref", *flags()).forward_images(li, center3d_override=vol)) for li in lists]
    m = new(weights, "bev", *flags())
    run = lambda: [snapshot(r) for r in m.forward_image_batches(iter(lists), center3d_override=vol)]
    control(harness, m, run, ref, [m.copy_stream], [(m.stream, s["h2d"]) for s in m.slots], "bev stream -> h2d, copy delayed")


def test_control_romp_read_back_waits_for_the_kernels(weights, models, harness):
    """ROMP _read_back: d2h_stream waits for the slot's done event before it reads the person count and rows."""
    batches, override, pads = romp_frames(4, 110)
    ref = frame_refs(models("romp", "ref", *flags()), "romp", batches, override, pads)
    m, co = new(weights, "romp", *flags()), torch.from_numpy(override).cuda()
    run = lambda: [snapshot(r) for r in m.forward_batches((torch.from_numpy(b).pin_memory() for b in batches), offsets=pads,
                                                          center_override=co)]
    control(harness, m, run, ref, [m.stream], [(m.d2h_stream, s["done"]) for s in m.slots], "romp d2h -> done, kernels delayed")
