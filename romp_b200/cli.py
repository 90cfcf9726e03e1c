"""Host layer of the ``romp`` and ``bev`` command lines: frames in, result files out, the GPU work in between done by the
batched entry points (``forward_image_batches`` / ``forward_video_batches``) on their two-slot pipeline.

The file formats are the reference's (simple_romp/romp/utils.py): the helpers below restate its IO functions, each
docstring citing the lines it restates.  Three threads of work overlap: a reader thread decodes the next list of frames,
the GPU runs the current one, and a small pool of writer threads encodes the PNG and npz files of the previous one.
Every queue between them is bounded, so memory does not grow with the length of a video.

``run_inputs`` (``--inputs``) runs many videos and frame folders in one process: a reader thread per open input, lists
of frames taken from the open inputs in round-robin order, and one writer pool for all of them.
"""
from __future__ import annotations

import collections
import os
import os.path as osp
import queue
import threading
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

READ_AHEAD = 2          # decoded lists the reader thread may hold beyond the one the GPU is given
WRITERS = 4             # writer threads encoding the PNG / npz files
INPUT_WRITERS = 8       # writer threads shared by every input of run_inputs (--inputs)
WRITE_BACKLOG = 256     # frames handed to the writers and not yet written
OPEN_INPUTS = 8         # inputs run_inputs reads at once (--open_inputs)


def encode_jpeg(image):
    """The bytes ``cv2.imwrite(path.jpg, image)`` writes: OpenCV's JPEG encoder with its default parameters."""
    ok, data = cv2.imencode(".jpg", image)
    if not ok:
        raise RuntimeError("cv2.imencode('.jpg') failed")
    return data


def output_paths(input_path, save_path):
    """(save_dir, path of the ``--save_video`` file) for ``-i input_path -o save_path``, after romp/utils.py:156-163: a
    save path without an extension is a directory and the video is named after the input, else it is named after the
    save path and lies beside it."""
    if len(osp.splitext(save_path)[1]) == 0:
        save_dir, name = save_path, osp.splitext(osp.basename(input_path))[0] + ".mp4"
    else:
        save_dir, name = osp.dirname(save_path), osp.splitext(osp.basename(save_path))[0] + ".mp4"
    return save_dir, osp.join(save_dir, name)


def _extract(video_path, frame_dir, decode):
    """video2frame (romp/utils.py:145-151) one frame at a time: frame i of the video's frame count goes to
    ``frame_dir/{i:08d}.jpg`` (a frame that fails to read is skipped and keeps its number free).  Yields (path, image)
    where image is the written JPEG decoded from memory, i.e. the pixels ``cv2.imread(path)`` gives, or None."""
    cap = cv2.VideoCapture(video_path)
    try:
        for frame_id in range(int(cap.get(cv2.CAP_PROP_FRAME_COUNT))):
            ok, frame = cap.read()
            if not ok:
                continue
            path = osp.join(frame_dir, "{:08d}.jpg".format(frame_id))
            data = encode_jpeg(frame)
            with open(path, "wb") as f:
                f.write(data.tobytes())
            yield path, cv2.imdecode(data, cv2.IMREAD_COLOR) if decode else None
    finally:
        cap.release()


def frame_source(input_path, save_path, decode=True):
    """The frames of ``-i input_path`` in order, after collect_frame_path (romp/utils.py:153-182).  Returns (an iterator
    of (frame path, BGR image or None), path of the ``--save_video`` file).

    A video file has its frames extracted to ``<save_dir>/<video name>_frames/{:08d}.jpg`` as the reference does, but as
    they are read: each frame is JPEG-encoded once, the bytes written, and the same bytes decoded from memory, so the
    model sees the recompressed frame the reference reads back with cv2.imread without a second read of the file.  A
    folder gives its files in ``sorted(os.listdir)`` order, read with cv2.imread.  With ``decode=False`` the images are
    None (only the files are produced)."""
    assert osp.exists(input_path), input_path + " does not exist"
    save_dir, video_save_path = output_paths(input_path, save_path)
    if osp.isfile(input_path):
        frame_dir = osp.join(save_dir, osp.splitext(osp.basename(input_path))[0] + "_frames")
        print(f"Extracting the frames of input {input_path} to {frame_dir}")
        os.makedirs(frame_dir, exist_ok=True)
        return _extract(input_path, frame_dir, decode), video_save_path
    assert osp.isdir(input_path), input_path + " is supposed to be a folder containing video frames"
    paths = [osp.join(input_path, name) for name in sorted(os.listdir(input_path))]
    return ((p, cv2.imread(p) if decode else None) for p in paths), video_save_path


def frame_codec(model):
    """The GPU JPEG codec (jpeg.FrameCodec) of ``model``'s device, built once per device, or None: for anything but a
    ROMP or BEV instance on a CUDA device, and when the codec's probe found that the installed OpenCV codes JPEG
    differently (the reason is printed once)."""
    from .bev import BEV
    from .main import ROMP
    if not isinstance(model, (ROMP, BEV)) or getattr(model.tdevice, "type", None) != "cuda":
        return None
    from .jpeg import FrameCodec
    key = model.tdevice.index
    with _CODECS_LOCK:
        if key not in _CODECS:
            codec = FrameCodec(model.tdevice)
            if not codec.usable:
                print(f"Extracting video frames on the CPU: {codec.reason}")
            _CODECS[key] = codec if codec.usable else None
        return _CODECS[key]


_CODECS, _CODECS_LOCK = {}, threading.Lock()


def _extract_gpu(codec, video_path, frame_dir, size):
    """``_extract`` with the JPEG round trip on the GPU: the frames are read with VideoCapture, and each list of ``size``
    goes through ``codec`` at once, which writes the same ``.jpg`` bytes and gives the same decoded frames.  Yields
    (path, decoded device frame, its host copy, event after which the device frame is complete)."""
    cap = cv2.VideoCapture(video_path)
    try:
        pending = []

        def flush():
            out, event = codec.run([f for _, f in pending])
            for (path, _), (data, dev, host) in zip(pending, out):
                with open(path, "wb") as f:
                    f.write(data)
                yield path, dev, host, event
            pending.clear()

        for frame_id in range(int(cap.get(cv2.CAP_PROP_FRAME_COUNT))):
            ok, frame = cap.read()
            if not ok:
                continue
            pending.append((osp.join(frame_dir, "{:08d}.jpg".format(frame_id)), frame))
            if len(pending) == size:
                yield from flush()
        if pending:
            yield from flush()
    finally:
        cap.release()


def model_frames(model, input_path, save_path):
    """``frame_source(input_path, save_path)`` for ``model``: a video file whose model has a usable GPU codec
    (``frame_codec``) has its frames extracted through it in lists of ``model.max_batch``, writing the same files and
    giving the same frames; items are then (path, device frame, host frame, event).  Everything else is
    ``frame_source``'s (path, image)."""
    codec = frame_codec(model) if osp.isfile(input_path) else None
    if codec is None:
        return frame_source(input_path, save_path)
    save_dir, video_save_path = output_paths(input_path, save_path)
    frame_dir = osp.join(save_dir, osp.splitext(osp.basename(input_path))[0] + "_frames")
    print(f"Extracting the frames of input {input_path} to {frame_dir}")
    os.makedirs(frame_dir, exist_ok=True)
    return _extract_gpu(codec, input_path, frame_dir, model.max_batch), video_save_path


def model_images(items):
    """The images the model gets for a list of frame items: a codec frame's device tensor, with the caller's current
    stream ordered after the codec's work (one event wait per list, no host sync), or the host image."""
    waited = set()
    for it in items:
        if len(it) == 4 and id(it[3]) not in waited:
            import torch
            torch.cuda.current_stream(it[1].device).wait_event(it[3])
            waited.add(id(it[3]))
    return [it[1] for it in items]


def saved_image(item):
    """The host image a frame item's PNG is written from."""
    return item[2] if len(item) == 4 else item[1]


def collect_frame_path(input_path, save_path):
    """collect_frame_path (romp/utils.py:153-182): extract a video's frames (or list a folder's) and return (frame paths,
    path of the ``--save_video`` file)."""
    frames, video_save_path = frame_source(input_path, save_path, decode=False)
    return [p for p, _ in frames], video_save_path


def read_ahead(frames, size, depth=READ_AHEAD):
    """Lists of up to ``size`` items of the iterator ``frames``, produced by a reader thread that stays at most ``depth``
    lists ahead of the consumer.  An exception in the reader is raised in the consumer; a consumer that stops early stops
    the reader."""
    q, stop, END = queue.Queue(maxsize=depth), threading.Event(), object()

    def put(item):
        while not stop.is_set():
            try:
                q.put(item, timeout=0.1)
                return True
            except queue.Full:
                pass
        return False

    def run():
        try:
            chunk = []
            for item in frames:
                chunk.append(item)
                if len(chunk) == size:
                    if not put(chunk):
                        return
                    chunk = []
            if chunk and not put(chunk):
                return
            put(END)
        except BaseException as e:          # handed to the consumer
            put(e)

    reader = threading.Thread(target=run, name="frame-reader", daemon=True)
    reader.start()
    try:
        while True:
            item = q.get()
            if item is END:
                return
            if isinstance(item, BaseException):
                raise item
            yield item
    finally:
        stop.set()
        reader.join()


class ResultSaver:
    """ResultSaver (romp/utils.py:43-86): where the result files of a frame go.

    - A save path without an extension is a directory.  In ``video`` mode, or with a directory, frame ``input_path`` is
      saved as ``<save_dir>/<input stem>.png``; in ``image`` mode with a file name, as that file.  A ``prefix`` appends
      ``_{prefix}`` to the stem.
    - ``<stem>.npz`` holds ``results=outputs`` and is written only when ``outputs`` is not None.
    - The PNG is always written.  It is ``outputs['rendered_image']`` when present; nothing here renders, so it is the
      input frame (``image``, or ``cv2.imread(input_path)`` when not given), as the reference writes it without a
      rendered image.

    ``writers`` > 0 encodes the files on that many threads, with at most WRITE_BACKLOG frames waiting; the files are the
    same as with the serial writer (``writers=0``).  A ``pool`` (WriterPool) instead shares its threads and its backlog
    with the other savers given it.  ``close()`` waits for every file and raises a writer's error."""

    def __init__(self, mode="image", save_path=None, save_npz=True, writers=0, pool=None):
        self.is_dir = len(osp.splitext(save_path)[1]) == 0
        self.mode = mode
        self.save_path = save_path
        self.save_npz = save_npz
        self.save_dir = save_path if self.is_dir else osp.dirname(save_path)
        if self.mode in ("image", "video"):
            os.makedirs(self.save_dir, exist_ok=True)
        if self.mode == "video":
            self.frame_save_paths = []
        self._own_pool = pool is None
        if pool is None:
            self._pool = ThreadPoolExecutor(writers, thread_name_prefix="result-writer") if writers > 0 else None
            self._backlog = threading.BoundedSemaphore(WRITE_BACKLOG)
        else:
            self._pool, self._backlog = pool.executor, pool.backlog
        self._pending = collections.deque()

    def path_of(self, input_path, prefix=None, img_ext=".png"):
        """The PNG path of frame ``input_path`` (romp/utils.py:56-63); its npz has the same stem."""
        if self.mode == "video" or self.is_dir:
            save_path = osp.join(self.save_dir, osp.splitext(osp.basename(input_path))[0]) + img_ext
        else:
            save_path = self.save_path
        if prefix is not None:
            save_path = osp.splitext(save_path)[0] + f"_{prefix}" + osp.splitext(save_path)[1]
        return save_path

    def __call__(self, outputs, input_path, prefix=None, img_ext=".png", image=None):
        save_path = self.path_of(input_path, prefix, img_ext)
        if self.mode == "video":
            self.frame_save_paths.append(save_path)
        if self._pool is None:
            self._write(outputs, input_path, save_path, image)
            return
        self._backlog.acquire()
        fut = self._pool.submit(self._write, outputs, input_path, save_path, image)
        fut.add_done_callback(lambda _: self._backlog.release())
        self._pending.append(fut)
        while self._pending and self._pending[0].done():
            self._pending.popleft().result()

    def _write(self, outputs, input_path, save_path, image):
        rendered = None
        if outputs is not None:
            rendered = outputs.pop("rendered_image", None)
            if self.save_npz:
                np.savez(osp.splitext(save_path)[0] + ".npz", results=outputs)
        if rendered is None:
            rendered = cv2.imread(input_path) if image is None else image
        if not cv2.imwrite(save_path, rendered):
            raise RuntimeError(f"cv2.imwrite failed for {save_path}")

    def close(self):
        """Wait until every file handed over has been written (a writer's error is raised here)."""
        while self._pending:
            self._pending.popleft().result()

    def save_video(self, save_path, frame_rate=24):
        """An ``mp4v`` video of the saved PNGs in order (romp/utils.py:78-85)."""
        self.close()
        if len(self.frame_save_paths) == 0:
            return
        height, width = cv2.imread(self.frame_save_paths[0]).shape[:2]
        writer = cv2.VideoWriter(save_path, cv2.VideoWriter_fourcc(*"mp4v"), frame_rate, (width, height))
        for frame_path in self.frame_save_paths:
            writer.write(cv2.imread(frame_path))
        writer.release()

    def __del__(self):
        if getattr(self, "_pool", None) is not None and self._own_pool:
            self._pool.shutdown(wait=True)


class WriterPool:
    """Writer threads and a backlog of at most WRITE_BACKLOG frames, shared by several ResultSavers (``run_inputs``), so
    that neither the thread count nor the memory held for writing grows with the number of inputs."""

    def __init__(self, writers):
        self.executor = ThreadPoolExecutor(writers, thread_name_prefix="input-writer")
        self.backlog = threading.BoundedSemaphore(WRITE_BACKLOG)

    def shutdown(self):
        self.executor.shutdown(wait=True)


def save_video_results(frame_save_paths):
    """save_video_results (romp/utils.py:88-110): ``video_results.npz`` beside the first frame, with ``results`` (each
    frame's result dict, keyed by its PNG's basename) and ``sequence_results`` (per track id: ``frame_id``, the frame's
    index in ``frame_save_paths``, and every key of the frame's results, as lists in frame order).  A frame without an
    npz (nobody detected) is left out; the reference stops with FileNotFoundError there."""
    video_results, sequence_results = {}, {}
    for frame_id, save_path in enumerate(frame_save_paths):
        npz_path = osp.splitext(save_path)[0] + ".npz"
        if not osp.exists(npz_path):
            continue
        frame_results = np.load(npz_path, allow_pickle=True)["results"][()]
        video_results[osp.basename(save_path)] = frame_results
        if "track_ids" not in frame_results:
            continue
        for subj, track_id in enumerate(frame_results["track_ids"]):
            seq = sequence_results.setdefault(track_id, {"frame_id": []})
            seq["frame_id"].append(frame_id)
            for key in frame_results:
                seq.setdefault(key, []).append(frame_results[key][subj])
    np.savez(osp.join(osp.dirname(frame_save_paths[0]), "video_results.npz"), results=video_results,
             sequence_results=sequence_results)


def run_frames(model, frames, saver, prefix=None, center_override=None):
    """Run ``frames`` (an iterable of (frame path, BGR image), or ``model_frames``' items) through ``model`` (a ROMP or BEV instance) in lists of
    ``model.max_batch`` and save every frame's result in order through ``saver``.

    ROMP with -t uses ``forward_video_batches`` (every frame on signal_ID 0), otherwise ``forward_image_batches``; BEV
    uses ``forward_image_batches`` with or without -t (wide frames go through crowd mode).  Each frame's result is what
    the per-frame loop of the reference's ``main()`` gives, within the documented equalities of those entry points.  A
    reader thread decodes list i+1 while the GPU runs list i and the writers save list i-1.  ``center_override``: the
    entry point's centre-map override, applied to every list (tests and measurement)."""
    from .main import ROMP
    in_flight = collections.deque()

    def images():
        for chunk in read_ahead(iter(frames), model.max_batch):
            in_flight.append(chunk)
            yield model_images(chunk)

    if isinstance(model, ROMP) and model.temporal is not None:
        results = model.forward_video_batches(images(), None, True, center_override)
    else:
        results = model.forward_image_batches(images(), True, center_override)
    for res in results:
        for item, out in zip(in_flight.popleft(), res):
            saver(out, item[0], prefix, image=saved_image(item))
    saver.close()


def run_video(model, args, prefix=None, center_override=None):
    """``--mode video`` (romp/main.py:187-196, bev/main.py:298-307): frames of ``args.input`` through ``run_frames``
    into ``args.save_path``, then ``video_results.npz`` and, with ``--save_video``, the mp4.  Returns the saver."""
    frames, video_save_path = model_frames(model, args.input, args.save_path)
    saver = ResultSaver("video", args.save_path, writers=WRITERS)
    run_frames(model, frames, saver, prefix, center_override)
    if saver.frame_save_paths:
        save_video_results(saver.frame_save_paths)
    if args.save_video:
        saver.save_video(video_save_path, frame_rate=args.frame_rate)
    return saver


# ----------------------------------------------------------------------------------------------------------------------
# --inputs: many videos and frame folders in one process


def input_dirs(inputs, save_path):
    """The output directory of every input of ``--inputs``: ``<save_path>/<input stem>``, where the input writes what
    ``-i input -o <save_path>/<input stem>`` writes.  Raises ValueError for a save path with an extension, a missing
    input, a stem with an extension (its directory would be taken for a file name) and two inputs with the same stem."""
    if not inputs:
        raise ValueError("--inputs: no input given")
    if len(osp.splitext(save_path)[1]) != 0:
        raise ValueError(f"--inputs writes one directory per input: -o {save_path} must be a directory (no extension)")
    dirs, seen = [], {}
    for p in inputs:
        if not osp.exists(p):
            raise ValueError(f"--inputs: {p} does not exist")
        stem = osp.splitext(osp.basename(osp.normpath(p)))[0]
        if not stem or len(osp.splitext(stem)[1]) != 0:
            raise ValueError(f"--inputs: the stem {stem!r} of {p} names its output directory and must not have an extension")
        if stem in seen:
            raise ValueError(f"--inputs: {seen[stem]} and {p} have the same stem {stem!r} and would write the same directory")
        seen[stem] = p
        dirs.append(osp.join(save_path, stem))
    return dirs


def check_inputs(args):
    """What ``--inputs`` refuses, before a model is built (ValueError): ``-i`` beside it, a mode but video, an
    ``--open_inputs`` below 1, the save paths and inputs of ``input_dirs``, and with -t a ``--video_streams`` below
    ``--open_inputs``.  With -t, ``--video_streams 0`` becomes ``--open_inputs``: one stream per open input."""
    if getattr(args, "inputs", None) is None:
        return
    if args.input is not None:
        raise ValueError("-i and --inputs cannot be used together")
    if args.mode != "video":
        raise ValueError(f"--inputs runs videos and frame folders: it needs --mode video, not --mode {args.mode}")
    if args.open_inputs < 1:
        raise ValueError(f"--open_inputs {args.open_inputs}: at least one input must be open")
    input_dirs(args.inputs, args.save_path)
    if args.temporal_optimize:
        if not args.video_streams:
            args.video_streams = args.open_inputs
        elif args.video_streams < args.open_inputs:
            raise ValueError(f"--video_streams {args.video_streams}: -t --inputs tracks each open input as its own stream, "
                             f"so it needs at least --open_inputs {args.open_inputs} streams (0 gives exactly that many)")


class InputsFailed(RuntimeError):
    """Inputs of ``run_inputs`` that failed; ``errors`` maps each one's path to its exception.  Every other input ran to
    the end."""

    def __init__(self, errors):
        self.errors = dict(errors)
        super().__init__(f"{len(self.errors)} of the inputs failed:\n" +
                         "\n".join(f"  {p}: {type(e).__name__}: {e}" for p, e in self.errors.items()))


class _Reader:
    """One input's frames in lists of up to ``size``, produced by a thread of its own that stays at most READ_AHEAD lists
    ahead (the bounded queue of ``read_ahead``) and taken one frame at a time without blocking.  ``frames()`` makes the
    frame iterator on that thread.  ``wake`` is set whenever a list, the end or an error is queued."""

    END = object()

    def __init__(self, frames, size, wake):
        self.q, self.stop, self.wake = queue.Queue(maxsize=READ_AHEAD), threading.Event(), wake
        self.head, self.done, self.error = collections.deque(), False, None
        self.thread = threading.Thread(target=self._run, args=(frames, size), name="input-reader", daemon=True)
        self.thread.start()

    def _put(self, item):
        while not self.stop.is_set():
            try:
                self.q.put(item, timeout=0.1)
                self.wake.set()
                return True
            except queue.Full:
                pass
        return False

    def _run(self, frames, size):
        it = None
        try:
            it, chunk = frames(), []
            for item in it:
                chunk.append(item)
                if len(chunk) == size:
                    if not self._put(chunk):
                        return
                    chunk = []
            if chunk and not self._put(chunk):
                return
            self._put(self.END)
        except BaseException as e:          # ends this input only
            self._put(e)
        finally:
            if hasattr(it, "close"):
                it.close()                  # a video's capture is released on this thread

    def ready(self):
        """Whether a frame can be taken now.  Notes the end of the input (``done``) and its error, once every frame read
        before them has been taken."""
        if not self.head and not self.done:
            try:
                item = self.q.get_nowait()
            except queue.Empty:
                return False
            if item is self.END:
                self.done = True
            elif isinstance(item, BaseException):
                self.done, self.error = True, item
            else:
                self.head.extend(item)
        return bool(self.head)

    def take(self):
        return self.head.popleft()

    def close(self):
        self.stop.set()
        self.thread.join()


def take_round_robin(sources, start, n):
    """Up to ``n`` items from ``sources`` (objects with ``ready()`` and ``take()``), one from each ready source in turn,
    beginning with ``sources[start]``, until n are taken or no source is ready.  Returns ([(source index, item)], the
    index to start from next time)."""
    out, k, pos, idle = [], len(sources), start, 0
    while len(out) < n and idle < k:
        s = sources[pos % k]
        if s.ready():
            out.append((pos % k, s.take()))
            idle = 0
        else:
            idle += 1
        pos += 1
    return out, pos % k if k else 0


class _Input:
    """One input of ``run_inputs``: where it writes, its reader and saver while it is open, and its frame counts."""

    def __init__(self, index, path, save_dir):
        self.index, self.path, self.save_dir = index, path, save_dir       # index: the input's signal_ID
        self.video_save_path = output_paths(path, save_dir)[1]
        self.reader = self.saver = self.error = None
        self.sent = self.back = 0     # frames in lists given to the model / whose results came back
        self.ended = False            # no more of its frames go to the model (read to the end, failed, or stopped)
        self.write_failed = False     # its saver failed: its remaining results are dropped


def _center_map_shape(model):
    from .main import ROMP
    return (1, 64, 64) if isinstance(model, ROMP) else (64, 128, 128)


def run_inputs(model, inputs, save_path, args, prefix=None, center_override=None):
    """``--mode video --inputs``: every input (a video file or a frame folder) through ``model`` (ROMP or BEV) in one
    process.  Input p writes into ``<save_path>/<stem of p>`` exactly what ``run_video`` writes for ``-i p -o
    <save_path>/<stem of p>`` on a fresh instance: the extracted frames, each frame's PNG and npz, ``video_results.npz``
    and with ``args.save_video`` the mp4.

    - ``args.open_inputs`` (K) inputs are open at once, each read and decoded by its own thread (``frame_source``) at
      most READ_AHEAD lists of ``max_batch`` frames ahead; the others open in list order as earlier ones end.
    - Each list of up to ``max_batch`` frames takes the ready frames of the open inputs in round-robin order, so a slow
      input does not hold back the others; each input's frames keep their order.  Input i has signal_ID i.
    - ROMP with -t runs ``forward_video_batches(..., signal_IDs)``, BEV with -t ``forward_image_batches(...,
      signal_IDs)``, both in stream mode with at least K streams; without -t both run ``forward_image_batches``.  Once an
      input's last list has been given to the model, ``reset_temporal(signal_ID)`` frees its stream before another input
      opens; once its results are back its files are finished.
    - The inputs' ResultSavers share INPUT_WRITERS writer threads and one backlog.
    - A reader's error, a writer's error or a failed BEV stream (StreamFailed) stops only its input; the files it wrote
      stay.  A failed stream loses the results of the lists in flight, so every other input with frames among them
      starts again from its first frame on a fresh stream (its files are written again, the same).  The others run to
      the end, every thread is joined, and then InputsFailed names the failed inputs.

    ``center_override``: callable (input index, frame index) -> centre map (ROMP [1,64,64], BEV's 3-D volume
    [64,128,128]) or None for a frame without one (BEV's crowd-mode frames); each list's maps are copied, in list order,
    into one device buffer on the model's stream ahead of the list's kernels (tests and measurement)."""
    from .streams import StreamFailed
    dirs = input_dirs(inputs, save_path)
    k_open = int(getattr(args, "open_inputs", OPEN_INPUTS))
    tracked = getattr(model, "temporal", None) not in (None, False)
    if tracked and getattr(model, "video_streams", 0) < k_open:
        raise ValueError(f"run_inputs with -t tracks each of {k_open} open inputs as its own stream: the model needs "
                         f"--video_streams >= {k_open}, it has {getattr(model, 'video_streams', 0)}")
    items = [_Input(i, osp.normpath(p), d) for i, (p, d) in enumerate(zip(inputs, dirs))]
    waiting, live, in_flight, sids = collections.deque(items), [], collections.deque(), collections.deque()
    wake, pool, turn = threading.Event(), WriterPool(INPUT_WRITERS), [0]
    co = None
    if center_override is not None:
        import torch
        co = torch.zeros((model.max_batch, *_center_map_shape(model)), device=getattr(model, "tdevice", "cpu"))

    def open_input(inp):
        inp.sent = inp.back = 0
        inp.ended, inp.error, inp.write_failed = False, None, False
        inp.saver = ResultSaver("video", inp.save_dir, pool=pool)
        inp.reader = _Reader(lambda: model_frames(model, inp.path, inp.save_dir)[0], model.max_batch, wake)
        live.append(inp)

    def stop(inp):
        if inp.reader is not None:
            inp.reader.close()
            inp.reader = None
        inp.ended = True

    def fail(inp, e):
        inp.error = inp.error or e
        stop(inp)

    def finish(inp):
        """An ended input whose results are all back: wait for its files, then video_results.npz and the mp4."""
        if not inp.ended or inp.back < inp.sent or inp.saver is None:
            return
        saver, inp.saver = inp.saver, None
        try:
            saver.close()
            if inp.error is None and saver.frame_save_paths:
                save_video_results(saver.frame_save_paths)
            if inp.error is None and getattr(args, "save_video", False):
                saver.save_video(inp.video_save_path, frame_rate=args.frame_rate)
        except Exception as e:
            inp.error = inp.error or e

    def put_override(batch):
        import torch
        maps = [m for m in (center_override(inp.index, t) for inp, t, _, _ in batch) if m is not None]
        if not maps:
            return
        if co.is_cuda:                      # after the previous list's kernels, before this one's
            model.stream.wait_stream(torch.cuda.current_stream(co.device))
            with torch.cuda.stream(model.stream):
                co[:len(maps)].copy_(torch.stack([torch.as_tensor(m).to(co.device) for m in maps]))
        else:
            co[:len(maps)].copy_(torch.stack([torch.as_tensor(m) for m in maps]))

    def lists():
        """The lists of images handed to the model; each one's (input, frame index, path, image) go to in_flight and
        its signal_IDs to sids."""
        while True:
            for inp in [x for x in live if x.ended]:       # its last list has been handed over: free its stream
                live.remove(inp)
                if tracked:
                    model.reset_temporal(inp.index)
                finish(inp)
            while waiting and len(live) < k_open:
                open_input(waiting.popleft())
            wake.clear()
            taken, turn[0] = take_round_robin([x.reader for x in live], turn[0], model.max_batch)
            for inp in live:
                if inp.reader.done and not inp.reader.head:
                    if inp.reader.error is not None:
                        inp.error = inp.reader.error
                    stop(inp)
            if taken:
                batch = []
                for k, item in taken:
                    batch.append((live[k], live[k].sent, item[0], item))
                    live[k].sent += 1
                in_flight.append(batch)
                sids.append([inp.index for inp, _, _, _ in batch])
                if co is not None:
                    put_override(batch)
                yield model_images([item for _, _, _, item in batch])
            elif not live and not waiting:
                return
            elif not any(x.ended for x in live):
                wake.wait(1.0)

    def signal_lists():
        while True:
            yield sids.popleft()

    def save(batch, res):
        for (inp, _, path, item), out in zip(batch, res):
            inp.back += 1
            if not inp.write_failed:
                try:
                    inp.saver(out, path, prefix, image=saved_image(item))
                except Exception as e:
                    inp.write_failed = True
                    fail(inp, e)
        for inp in {x for x, _, _, _ in batch}:
            finish(inp)

    def recover(err):
        """A failed stream: its input stops; the other inputs in the lost lists start again (see above)."""
        lost = {inp for batch in in_flight for inp, _, _, _ in batch}
        in_flight.clear()
        sids.clear()
        failed = [inp for inp in items if inp.index in set(err.signal_IDs)]
        if not tracked or not failed:
            raise err
        again = []
        for inp in items:
            if inp not in failed and inp not in lost:
                continue
            if inp in live:
                live.remove(inp)
            model.reset_temporal(inp.index)
            if inp in failed:
                fail(inp, err)
                inp.back = inp.sent
                finish(inp)
                continue
            stop(inp)
            saver, inp.saver = inp.saver, None
            try:
                saver.close()
            except Exception as e:
                fail(inp, e)
                continue
            again.append(inp)
        waiting.extendleft(reversed(again))

    try:
        while True:
            if tracked and hasattr(model, "forward_video_batches"):
                results = model.forward_video_batches(lists(), signal_lists(), True, co)
            elif tracked:
                results = model.forward_image_batches(lists(), True, co, signal_lists())
            else:
                results = model.forward_image_batches(lists(), True, co)
            try:
                for res in results:
                    save(in_flight.popleft(), res)
                break
            except StreamFailed as e:
                recover(e)
    finally:
        for inp in items:
            if inp.reader is not None:
                inp.reader.close()
        pool.shutdown()
    errors = {inp.path: inp.error for inp in items if inp.error is not None}
    if errors:
        raise InputsFailed(errors)


def run_inputs_command(model, args, prefix=None):
    """``--inputs`` of the command lines: ``run_inputs`` into ``args.save_path``; a failed input makes the command exit
    with status 1, naming every failed input."""
    try:
        run_inputs(model, args.inputs, args.save_path, args, prefix)
    except InputsFailed as e:
        raise SystemExit(str(e))
