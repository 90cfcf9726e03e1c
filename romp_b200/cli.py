"""Host layer of the ``romp`` and ``bev`` command lines: frames in, result files out, the GPU work in between done by the
batched entry points (``forward_image_batches`` / ``forward_video_batches``) on their two-slot pipeline.

The file formats are the reference's (simple_romp/romp/utils.py): the helpers below restate its IO functions, each
docstring citing the lines it restates.  Three threads of work overlap: a reader thread decodes the next list of frames,
the GPU runs the current one, and a small pool of writer threads encodes the PNG and npz files of the previous one.
Every queue between them is bounded, so memory does not grow with the length of a video.
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
WRITE_BACKLOG = 256     # frames handed to the writers and not yet written


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
    same as with the serial writer (``writers=0``).  ``close()`` waits for every file and raises a writer's error."""

    def __init__(self, mode="image", save_path=None, save_npz=True, writers=0):
        self.is_dir = len(osp.splitext(save_path)[1]) == 0
        self.mode = mode
        self.save_path = save_path
        self.save_npz = save_npz
        self.save_dir = save_path if self.is_dir else osp.dirname(save_path)
        if self.mode in ("image", "video"):
            os.makedirs(self.save_dir, exist_ok=True)
        if self.mode == "video":
            self.frame_save_paths = []
        self._pool = ThreadPoolExecutor(writers, thread_name_prefix="result-writer") if writers > 0 else None
        self._backlog = threading.BoundedSemaphore(WRITE_BACKLOG)
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
        if getattr(self, "_pool", None) is not None:
            self._pool.shutdown(wait=True)


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
    """Run ``frames`` (an iterable of (frame path, BGR image)) through ``model`` (a ROMP or BEV instance) in lists of
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
            yield [image for _, image in chunk]

    if isinstance(model, ROMP) and model.temporal is not None:
        results = model.forward_video_batches(images(), None, True, center_override)
    else:
        results = model.forward_image_batches(images(), True, center_override)
    for res in results:
        for (path, image), out in zip(in_flight.popleft(), res):
            saver(out, path, prefix, image=image)
    saver.close()


def run_video(model, args, prefix=None, center_override=None):
    """``--mode video`` (romp/main.py:187-196, bev/main.py:298-307): frames of ``args.input`` through ``run_frames``
    into ``args.save_path``, then ``video_results.npz`` and, with ``--save_video``, the mp4.  Returns the saver."""
    frames, video_save_path = frame_source(args.input, args.save_path)
    saver = ResultSaver("video", args.save_path, writers=WRITERS)
    run_frames(model, frames, saver, prefix, center_override)
    if saver.frame_save_paths:
        save_video_results(saver.frame_save_paths)
    if args.save_video:
        saver.save_video(video_save_path, frame_rate=args.frame_rate)
    return saver
