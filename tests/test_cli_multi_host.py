"""``--inputs`` (romp_b200/cli.py ``run_inputs``) on the CPU, with fake models that record every call and return results
keyed by (input, frame index): each input's files equal those of a single-input ``run_video`` on a fresh fake, whatever
the scheduling; the order of each input's frames, round-robin lists, the number of open inputs and live streams, the
resets, bounded readers, failures that stop only their own input, no thread left behind, and the argument errors."""
import os
import threading
import time
import types

import cv2
import numpy as np
import pytest
import torch

from romp_b200 import cli
from romp_b200.streams import StreamFailed

LENGTHS = [9, 0, 14, 1, 23]                 # frames per input; input 1 is an empty folder


def key_image(i, t):
    img = np.zeros((6, 8, 3), np.uint8)
    img[0, 0] = (i, t % 256, t // 256)
    img[1:, :] = (7 * i + 3 * t) % 256
    return img


def image_key(img):
    return int(img[0, 0, 0]), int(img[0, 0, 1]) + 256 * int(img[0, 0, 2])


class FakeModel:
    """``forward_image_batches`` (BEV's signature) on the two-slot pattern of the real entry points: list i+1 is pulled
    before the result of list i is given.  A frame's result is keyed by its input and frame index (and signal_ID with
    -t); every fifth frame has nobody.  ``fail``: (input, frame) whose list's read-back raises StreamFailed."""

    def __init__(self, max_batch=4, temporal=False, video_streams=0, fail=None, delay=0.0, on_list=None):
        self.max_batch, self.temporal, self.video_streams = max_batch, temporal, video_streams
        self.fail, self.delay, self.on_list = fail, delay, on_list
        self.calls, self.live, self.max_live = [], set(), 0

    def reset_temporal(self, signal_ID=None):
        self.calls.append(("reset", signal_ID))
        self.live.discard(signal_ID)

    def _results(self, batches, sid_iter, co):
        pending = None
        for images in batches:
            keys = [image_key(x) for x in images]
            sids = list(next(sid_iter)) if sid_iter is not None else [0] * len(keys)     # run_frames: signal 0
            if self.temporal:
                assert sid_iter is None or sids == [i for i, _ in keys]
                self.live |= set(sids)
                self.max_live = max(self.max_live, len(self.live))
                assert len(self.live) <= self.video_streams
            self.calls.append(("list", keys))
            if self.on_list is not None:
                self.on_list(self, keys)
            time.sleep(self.delay)
            res = []
            for k, (i, t) in enumerate(keys):
                r = None if t % 5 == 4 else dict(frame=np.array([i, t], np.int64), cam=np.full((2, 3), i + t / 100, np.float32))
                if r is not None and co is not None:
                    r["co"] = np.array([float(co[k].flatten()[0])])
                if r is not None and self.temporal:
                    r["track_ids"] = np.array([1, 2], np.int32)
                res.append(r)
            if pending is not None:
                yield self._finish(*pending)
            pending = (keys, res)
        if pending is not None:
            yield self._finish(*pending)

    def _finish(self, keys, res):
        if self.fail in keys:
            self.calls.append(("raised", None))
            raise StreamFailed(f"stream of signal_ID {self.fail[0]} is full", [self.fail[0]])
        return res

    def forward_image_batches(self, batches, to_numpy=True, center_override=None, signal_IDs=None):
        return self._results(batches, None if signal_IDs is None else iter(signal_IDs), center_override)


class FakeVideoModel(FakeModel):
    """ROMP's signatures: ``forward_image_batches(batches, to_numpy, center_override)`` and, with -t,
    ``forward_video_batches(batches, signal_IDs, to_numpy, center_override)``."""

    def forward_image_batches(self, batches, to_numpy=True, center_override=None):
        return self._results(batches, None, center_override)

    def forward_video_batches(self, batches, signal_IDs=None, to_numpy=True, center_override=None):
        return self._results(batches, iter(signal_IDs), center_override)


def make_inputs(root, lengths=LENGTHS):
    paths = []
    for i, n in enumerate(lengths):
        d = os.path.join(root, f"clip{i}")
        os.makedirs(d)
        for t in range(n):
            assert cv2.imwrite(os.path.join(d, f"{t:05d}.png"), key_image(i, t))
        paths.append(d)
    return paths


def args_of(**kw):
    a = dict(open_inputs=cli.OPEN_INPUTS, save_video=False, frame_rate=24)
    a.update(kw)
    return types.SimpleNamespace(**a)


def read(p):
    with open(p, "rb") as f:
        return f.read()


def same_value(a, b):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b)
        for k in a:
            same_value(a[k], b[k])
    elif isinstance(a, list):
        assert isinstance(b, list) and len(a) == len(b)
        for x, y in zip(a, b):
            same_value(x, y)
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y)


def same_tree(d1, d2):
    """Same files, recursively; PNG and JPEG bytes equal; npz files with equal arrays."""
    names = sorted(os.listdir(d1))
    assert names == sorted(os.listdir(d2)), (d1, names, sorted(os.listdir(d2)))
    for name in names:
        a, b = os.path.join(d1, name), os.path.join(d2, name)
        if os.path.isdir(a):
            same_tree(a, b)
        elif name.endswith(".npz"):
            x, y = np.load(a, allow_pickle=True), np.load(b, allow_pickle=True)
            assert sorted(x.files) == sorted(y.files)
            for k in x.files:
                same_value(x[k][()], y[k][()])
        else:
            assert read(a) == read(b), a


def single_runs(tmp_path, paths, make, prefix, skip=()):
    """Every input through run_video on a fresh model, into ref/<stem>."""
    ref = str(tmp_path / "ref")
    for i, p in enumerate(paths):
        if i in skip:
            continue
        out = os.path.join(ref, os.path.basename(p))
        cli.run_video(make(), types.SimpleNamespace(input=p, save_path=out, save_video=False, frame_rate=24), prefix)
    return ref


def pool_threads():
    return [t for t in threading.enumerate() if t.name.startswith(("input-reader", "input-writer")) and t.is_alive()]


@pytest.fixture
def counted_sources(monkeypatch):
    """frame_source wrapped to count the inputs open at once and the frames read."""
    stats = dict(open=0, max_open=0, read=0, lock=threading.Lock())
    real = cli.frame_source

    def source(path, save_path, decode=True):
        frames, vpath = real(path, save_path, decode)

        def gen():
            with stats["lock"]:
                stats["open"] += 1
                stats["max_open"] = max(stats["max_open"], stats["open"])
            try:
                for f in frames:
                    with stats["lock"]:
                        stats["read"] += 1
                    yield f
            finally:
                with stats["lock"]:
                    stats["open"] -= 1
        return gen(), vpath

    monkeypatch.setattr(cli, "frame_source", source)
    return stats


def check_order_and_resets(model, lengths, tracked):
    """Each input's frames go to the model in order, each once; with -t each input is reset once, after its last list
    and before any list of an input opened later."""
    lists = [keys for kind, keys in model.calls if kind == "list"]
    for i, n in enumerate(lengths):
        assert [t for keys in lists for j, t in keys if j == i] == list(range(n))
    for keys in lists:
        seen = {}
        for i, t in keys:
            assert t > seen.get(i, -1)
            seen[i] = t
    resets = [sid for kind, sid in model.calls if kind == "reset"]
    if not tracked:
        assert resets == []
        return
    assert sorted(resets) == list(range(len(lengths)))
    for i in range(len(lengths)):
        at = model.calls.index(("reset", i))
        assert all(j != i for kind, keys in model.calls[at:] if kind == "list" for j, _ in keys)


@pytest.mark.parametrize("kind", ["romp", "bev"])
@pytest.mark.parametrize("tracked", [False, True], ids=["plain", "tracked"])
@pytest.mark.parametrize("open_inputs,max_batch", [(2, 3), (3, 8), (8, 4)])
def test_each_input_equals_a_single_input_run(tmp_path, counted_sources, kind, tracked, open_inputs, max_batch):
    cls = FakeVideoModel if kind == "romp" else FakeModel
    paths = make_inputs(str(tmp_path / "in"))
    prefix = None if kind == "romp" else "_2_0.12"
    model = cls(max_batch, tracked, open_inputs if tracked else 0, delay=0.002)
    out = str(tmp_path / "out")
    cli.run_inputs(model, paths, out, args_of(open_inputs=open_inputs), prefix)
    assert pool_threads() == []
    assert counted_sources["max_open"] <= open_inputs
    if tracked:
        assert model.max_live <= open_inputs
    check_order_and_resets(model, LENGTHS, tracked)
    lists = [keys for kind_, keys in model.calls if kind_ == "list"]
    assert all(1 <= len(keys) <= max_batch for keys in lists)
    ref = single_runs(tmp_path, paths, lambda: cls(max_batch, tracked, 1 if tracked else 0), prefix)
    same_tree(out, ref)
    assert sorted(os.listdir(out)) == [f"clip{i}" for i in range(len(LENGTHS))]
    assert not os.path.exists(os.path.join(out, "clip1", "video_results.npz"))         # an empty input: no results


class Source:
    def __init__(self, items, ready=True):
        self.items, self.on = list(items), ready

    def ready(self):
        return self.on and bool(self.items)

    def take(self):
        return self.items.pop(0)


def test_round_robin_lists():
    s = [Source("abc"), Source("de"), Source("fghij")]
    out, nxt = cli.take_round_robin(s, 0, 6)
    assert [x for _, x in out] == list("adfbeg") and nxt == 0
    out, nxt = cli.take_round_robin(s, nxt, 6)
    assert [x for _, x in out] == list("chij") and [k for k, _ in out] == [0, 2, 2, 2]
    held = [Source("ab", ready=False), Source("cd"), Source("ef")]
    out, nxt = cli.take_round_robin(held, 1, 3)
    assert [x for _, x in out] == list("ced") and nxt == 2          # the held source is passed over
    held[0].on = True
    out, _ = cli.take_round_robin(held, nxt, 8)
    assert [x for _, x in out] == list("fab")
    assert cli.take_round_robin([], 0, 4) == ([], 0)
    assert cli.take_round_robin([Source("")], 0, 4) == ([], 0)


def test_held_back_reader_does_not_stall_the_others(tmp_path, monkeypatch):
    """Input 0's reader is held until the model has had every frame of the others: their lists go on without it."""
    paths = make_inputs(str(tmp_path / "in"))
    others = sum(LENGTHS[1:])
    release = threading.Event()
    real = cli.frame_source

    def source(path, save_path, decode=True):
        frames, vpath = real(path, save_path, decode)
        if path.endswith("clip0"):
            def held():
                assert release.wait(60), "the other inputs did not get through while input 0 was held"
                yield from frames
            return held(), vpath
        return frames, vpath

    def on_list(model, keys):
        got = sum(len([1 for i, _ in k if i != 0]) for kind, k in model.calls if kind == "list")
        if got == others:
            release.set()

    monkeypatch.setattr(cli, "frame_source", source)
    model = FakeModel(4, True, 8, on_list=on_list)
    out = str(tmp_path / "out")
    cli.run_inputs(model, paths, out, args_of(), "_2_0.12")
    lists = [keys for kind, keys in model.calls if kind == "list"]
    first0 = next(n for n, keys in enumerate(lists) if any(i == 0 for i, _ in keys))
    assert sum(len([1 for i, _ in k if i != 0]) for k in lists[:first0]) == others
    check_order_and_resets(model, LENGTHS, True)
    monkeypatch.setattr(cli, "frame_source", real)
    same_tree(out, single_runs(tmp_path, paths, lambda: FakeModel(4, True, 1), "_2_0.12"))


def test_round_robin_when_every_reader_is_ahead(tmp_path, monkeypatch):
    """Readers held until all three have a list queued: then the lists alternate between them frame by frame."""
    paths = make_inputs(str(tmp_path / "in"), [8, 8, 8])
    barrier = threading.Barrier(3)
    real = cli.frame_source

    def source(path, save_path, decode=True):
        frames, vpath = real(path, save_path, decode)

        def gen():
            items = list(frames)
            barrier.wait(30)
            yield from items
        return gen(), vpath

    def on_list(model, keys):
        if len([k for kind, k in model.calls if kind == "list"]) == 1:
            time.sleep(0.2)             # every reader queues its lists

    monkeypatch.setattr(cli, "frame_source", source)
    orig = cli.take_round_robin
    calls = []

    def rr(sources, start, n):
        if not calls:                   # the first list: wait until every reader has one queued
            deadline = time.time() + 30
            while not all(s.q.qsize() or s.head for s in sources) and time.time() < deadline:
                time.sleep(0.01)
        calls.append(1)
        return orig(sources, start, n)

    monkeypatch.setattr(cli, "take_round_robin", rr)
    model = FakeModel(6, False, 0, on_list=on_list)
    cli.run_inputs(model, paths, str(tmp_path / "out"), args_of(open_inputs=3))
    lists = [keys for kind, keys in model.calls if kind == "list"]
    assert [i for i, _ in lists[0]] == [0, 1, 2, 0, 1, 2]
    assert [i for i, _ in lists[1]] == [0, 1, 2, 0, 1, 2]


def test_readers_stay_bounded(tmp_path, counted_sources):
    """A slow model: the frames read and not yet given to it stay within K x (READ_AHEAD + 2) lists."""
    lengths = [60, 60, 60]
    paths = make_inputs(str(tmp_path / "in"), lengths)
    B, K = 4, 3
    bound = K * (cli.READ_AHEAD + 2) * B
    ahead = []

    def on_list(model, keys):
        given = sum(len(k) for kind, k in model.calls if kind == "list")
        ahead.append(counted_sources["read"] - given)

    model = FakeModel(B, False, 0, delay=0.01, on_list=on_list)
    cli.run_inputs(model, paths, str(tmp_path / "out"), args_of(open_inputs=K))
    assert max(ahead) <= bound and max(ahead) > B          # the readers did run ahead, within the bound


def test_a_failing_reader_stops_only_its_input(tmp_path, monkeypatch):
    paths = make_inputs(str(tmp_path / "in"))
    real = cli.frame_source

    def source(path, save_path, decode=True):
        frames, vpath = real(path, save_path, decode)
        if path.endswith("clip2"):
            def broken():
                for t, f in enumerate(frames):
                    if t == 6:
                        raise OSError("unreadable frame")
                    yield f
            return broken(), vpath
        return frames, vpath

    monkeypatch.setattr(cli, "frame_source", source)
    model = FakeVideoModel(4, True, 3)
    out = str(tmp_path / "out")
    with pytest.raises(cli.InputsFailed, match="unreadable frame") as e:
        cli.run_inputs(model, paths, out, args_of(open_inputs=3))
    assert list(e.value.errors) == [paths[2]]
    assert pool_threads() == []
    assert ("reset", 2) in model.calls
    monkeypatch.setattr(cli, "frame_source", real)
    ref = single_runs(tmp_path, paths, lambda: FakeVideoModel(4, True, 1), None, skip=(2,))
    for i in (0, 1, 3, 4):
        same_tree(os.path.join(out, f"clip{i}"), os.path.join(ref, f"clip{i}"))
    # the frames read before the error (its reader's first list; the list it was building is lost) are saved
    written = sorted(os.listdir(os.path.join(out, "clip2")))
    assert "video_results.npz" not in written and [n for n in written if n.endswith(".png")] == [f"{t:05d}.png" for t in range(4)]


def test_a_failing_stream_stops_only_its_input(tmp_path):
    """A full track table in input 2's stream (frame 6): input 2 stops and is reset; the inputs whose lists were lost
    start again, and every other input's files equal a single-input run."""
    paths = make_inputs(str(tmp_path / "in"))
    model = FakeModel(4, True, 3, fail=(2, 6))
    out = str(tmp_path / "out")
    with pytest.raises(cli.InputsFailed, match="signal_ID 2") as e:
        cli.run_inputs(model, paths, out, args_of(open_inputs=3), "_2_0.12")
    assert list(e.value.errors) == [paths[2]]
    assert pool_threads() == []
    assert model.max_live <= 3
    assert ("reset", 2) in model.calls
    after = model.calls[model.calls.index(("raised", None)):]
    assert not any(i == 2 for kind, keys in after if kind == "list" for i, _ in keys)
    ref = single_runs(tmp_path, paths, lambda: FakeModel(4, True, 1), "_2_0.12", skip=(2,))
    for i in (0, 1, 3, 4):
        same_tree(os.path.join(out, f"clip{i}"), os.path.join(ref, f"clip{i}"))
    assert not os.path.exists(os.path.join(out, "clip2", "video_results.npz"))


def test_no_thread_is_left_after_a_model_error(tmp_path):
    paths = make_inputs(str(tmp_path / "in"))

    def boom(model, keys):
        if len([1 for kind, _ in model.calls if kind == "list"]) == 3:
            raise RuntimeError("device lost")

    with pytest.raises(RuntimeError, match="device lost"):
        cli.run_inputs(FakeModel(4, False, 0, on_list=boom), paths, str(tmp_path / "out"), args_of(open_inputs=2))
    assert pool_threads() == []


def test_center_override_per_frame(tmp_path):
    """The hook's map of (input, frame) reaches that frame, wherever the scheduler puts it in a list."""
    paths = make_inputs(str(tmp_path / "in"))
    hook = lambda i, t: torch.full((64, 128, 128), float(1000 * i + t))
    out = str(tmp_path / "out")
    cli.run_inputs(FakeModel(4, False, 0), paths, out, args_of(open_inputs=3), None, hook)
    n = 0
    for i, length in enumerate(LENGTHS):
        for t in range(length):
            npz = os.path.join(out, f"clip{i}", f"{t:05d}.npz")
            if t % 5 != 4:
                assert float(np.load(npz, allow_pickle=True)["results"][()]["co"][0]) == 1000 * i + t
                n += 1
    assert n > 30


def test_save_video_per_input(tmp_path):
    paths = make_inputs(str(tmp_path / "in"), [5, 3])
    out = str(tmp_path / "out")
    cli.run_inputs(FakeModel(4, False, 0), paths, out, args_of(save_video=True, frame_rate=12))
    for i, n in enumerate([5, 3]):
        cap = cv2.VideoCapture(os.path.join(out, f"clip{i}", f"clip{i}.mp4"))
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == n
        cap.release()


def test_video_input_extracts_its_frames(tmp_path):
    """A video file: its frames are extracted into <out>/<stem>/<stem>_frames, as -i <video> -o <out>/<stem> does."""
    video = str(tmp_path / "cam.avi")
    vw = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*"MJPG"), 24, (64, 48))
    rs = np.random.RandomState(0)
    for _ in range(6):
        vw.write(rs.randint(0, 256, (48, 64, 3)).astype(np.uint8))
    vw.release()

    class Plain(FakeModel):
        def _results(self, batches, sid_iter, co):
            for images in batches:
                yield [dict(mean=np.array([float(x.mean())])) for x in images]

    out, ref = str(tmp_path / "out"), str(tmp_path / "ref" / "cam")
    cli.run_inputs(Plain(4), [video], out, args_of())
    cli.run_video(Plain(4), types.SimpleNamespace(input=video, save_path=ref, save_video=False, frame_rate=24))
    same_tree(os.path.join(out, "cam"), ref)
    assert len(os.listdir(os.path.join(out, "cam", "cam_frames"))) == 6


def test_run_inputs_refuses_too_few_streams(tmp_path):
    paths = make_inputs(str(tmp_path / "in"), [2, 2])
    with pytest.raises(ValueError, match="video_streams >= 4"):
        cli.run_inputs(FakeModel(4, True, 2), paths, str(tmp_path / "out"), args_of(open_inputs=4))


def argument_cases(tmp_path):
    a, b = str(tmp_path / "a.mp4"), str(tmp_path / "x" / "a")
    os.makedirs(b)
    open(a, "wb").close()
    out = str(tmp_path / "out")
    return [
        (["--mode", "video", "-i", a, "--inputs", b, "-o", out], "-i and --inputs cannot be used together"),
        (["--inputs", b, "-o", out], "needs --mode video"),
        (["--mode", "video", "--inputs", b, str(tmp_path / "missing.mp4"), "-o", out], "does not exist"),
        (["--mode", "video", "--inputs", a, b, "-o", out], "have the same stem 'a'"),
        (["--mode", "video", "--inputs", b, "-o", str(tmp_path / "out.mp4")], "must be a directory"),
        (["--mode", "video", "-t", "--inputs", b, "--open_inputs", "4", "--video_streams", "3", "-o", out],
         "--video_streams 3"),
        (["--mode", "video", "--inputs", b, "--open_inputs", "0", "-o", out], "--open_inputs 0"),
    ]


@pytest.mark.parametrize("module", ["romp.main", "bev.main"])
def test_argument_errors_come_before_a_model(tmp_path, module):
    import importlib
    main = importlib.import_module(module).main
    for argv, message in argument_cases(tmp_path):
        with pytest.raises(ValueError, match=message.replace("(", r"\(").replace(")", r"\)")):
            main(argv + ["--model_path", "/nonexistent/model.pth"])


@pytest.mark.parametrize("module", ["romp.main", "bev.main"])
def test_video_streams_default_to_open_inputs(tmp_path, module):
    import importlib
    m = importlib.import_module(module)
    settings = m.romp_settings if module == "romp.main" else m.bev_settings
    d = str(tmp_path / "clip")
    os.makedirs(d)
    s = settings(["--mode", "video", "-t", "--inputs", d, "--open_inputs", "5", "-o", str(tmp_path / "out")])
    m.main.__globals__["check_cli"](s)
    assert s.video_streams == 5
    s = settings(["--mode", "video", "--inputs", d, "-o", str(tmp_path / "out")])
    m.main.__globals__["check_cli"](s)
    assert s.video_streams == 0 and s.open_inputs == cli.OPEN_INPUTS
