"""Stream mode of the video paths (``--video_streams N`` with ``-t``): host bookkeeping of which stream index each
``signal_ID`` holds.

Each distinct signal_ID is an independent video with its own tracker, track ids (from 1) and One-Euro filters, kept in
device memory at its stream index (csrc/track.cu, csrc/romp_track.cu); one kernel launch steps every stream of a batch
in parallel.  A new signal_ID takes the lowest free index, which is reset on the model's stream before the batch's
kernel; ``reset_temporal(signal_ID)`` frees it.  There is no eviction: a batch that would make more than N streams live
is refused before anything is enqueued.
"""
from __future__ import annotations

MAX_VIDEO_STREAMS = 1024       # B200ROMP_MAX_VIDEO_STREAMS, include/b200romp.h


class StreamFailed(RuntimeError):
    """Streams of a batch could not be tracked (BEV: a full track table); ``signal_IDs`` lists their signal_IDs.  The
    other streams of the batch were tracked; each failed one does nothing until ``reset_temporal(signal_ID)``."""

    def __init__(self, message, signal_IDs):
        super().__init__(message)
        self.signal_IDs = list(signal_IDs)


def check_video_streams(settings, temporal):
    """--video_streams of ``settings``, validated: 0 (one tracker per instance) or 1..MAX_VIDEO_STREAMS with -t."""
    n = int(getattr(settings, "video_streams", 0) or 0)
    if n < 0 or n > MAX_VIDEO_STREAMS:
        raise ValueError(f"--video_streams {n}: must be in [0, {MAX_VIDEO_STREAMS}]")
    if n and not temporal:
        raise ValueError("--video_streams tracks videos: it needs -t/--temporal_optimize")
    return n


def check_streams(live, signal_IDs, n):
    """Raise ValueError when the signal_IDs not in ``live`` (signal_ID -> stream index) would make more than n streams."""
    new = set(signal_IDs) - set(live)
    if len(live) + len(new) > n:
        raise ValueError(f"--video_streams {n}: this batch would make {len(live) + len(new)} streams live; call "
                         "reset_temporal(signal_ID) for the streams that ended")


def stream_indices(live, signal_IDs, n, reset):
    """The stream index of every signal_ID; a new signal_ID takes the lowest free index, which ``reset(index)`` resets
    (on the model's stream, before the batch's kernel).  ``live`` (signal_ID -> index) is updated in place."""
    check_streams(live, signal_IDs, n)
    out = []
    for sid in signal_IDs:
        if sid not in live:
            used = set(live.values())
            k = next(k for k in range(n) if k not in used)
            reset(k)
            live[sid] = k
        out.append(live[sid])
    return out
