"""Temporal path of ``ROMP.forward`` (``--temporal_optimize``; simple_romp/romp/main.py:117-157).

Per frame, between the parse and the SMPL forward: every detection is associated with a track, and the track's One-Euro
filters smooth (smpl_thetas, smpl_betas, cam).  The filters run on the device (``b200romp_one_euro_smooth``,
csrc/temporal.cu - state per track in device memory); this module is the host-side bookkeeping: which filter slot each
person uses.

* ``--show_largest`` (main.py:128-134): no tracker - the person with the largest cam scale uses ONE filter set per signal.
* otherwise the reference associates detections with ``norfair.Tracker(distance_function=euclidean_distance,
  distance_threshold=200)`` on the points ``cam[[2,1]] * 512`` and takes, for each detection, the id of the nearest
  tracked object (utils.py:275-280).  ``norfair`` is a third-party package that is neither vendored in the reference nor
  installed here (the reference pip-installs it on demand, main.py:120-125), so its Kalman-filter tracker is NOT
  restated: ``NearestCenterTracker`` below is a plain nearest-neighbour association with the same distance threshold -
  "parity unpinned" for the ids, which remain so; the filter recurrence is the reference's in both modes: --show_largest
  differentiates against the previous raw sample (tests/golden/one_euro.npz), the tracked mode - where the reference
  smooths views of the output rows and writes the results back into them (main.py:152-154) - against the previous
  smoothed value of body pose, betas and cam (tests/golden/one_euro_tracked.npz); ``b200romp_one_euro_smooth`` takes
  the mode as its ``tracked`` argument.
"""
from __future__ import annotations

import numpy as np

MAX_TRACKS_PER_SIGNAL = 64


class NearestCenterTracker:
    """id of the nearest live track within ``distance_threshold`` (same metric / threshold as the reference's norfair
    set-up), else a new id; tracks unseen for ``max_age`` frames are dropped."""

    def __init__(self, distance_threshold=200.0, max_age=30):
        self.thr, self.max_age = float(distance_threshold), int(max_age)
        self.tracks = {}              # id -> [point(2,), age]
        self.next_id = 1

    def update(self, points):
        ids, fresh = [], []
        for p in np.asarray(points, np.float64).reshape(-1, 2):
            best, bd = None, self.thr
            for tid, (q, _) in self.tracks.items():
                d = float(np.linalg.norm(p - q))
                if d < bd:
                    best, bd = tid, d
            if best is None:
                best = self.next_id
                self.next_id += 1
                fresh.append(best)
            self.tracks[best] = [p, 0]
            ids.append(best)
        for tid in list(self.tracks):
            if tid not in ids:
                self.tracks[tid][1] += 1
                if self.tracks[tid][1] > self.max_age:
                    del self.tracks[tid]
        return ids, fresh


class TemporalState:
    """Filter-slot bookkeeping for all signals of one ROMP instance (OE_filters of main.py:118, check_filter_state
    utils.py:248-256)."""

    def __init__(self, show_largest: bool, max_signals: int = 4):
        self.show_largest = bool(show_largest)
        self.max_signals = max_signals
        self.signals = {}             # signal_ID -> (base slot, tracker, {track id -> slot})

    @property
    def n_slots(self):
        return self.max_signals * MAX_TRACKS_PER_SIGNAL

    def assign(self, cams, signal_ID):
        """cams [N,3] (host) -> (slots int32 [N] (-1 = not smoothed), track ids int32 [N] or None, slots to reset)."""
        if signal_ID not in self.signals:
            if len(self.signals) >= self.max_signals:
                self.signals.pop(next(iter(self.signals)))
            used = {b for b, _, _ in self.signals.values()}
            base = next(b for b in range(0, self.n_slots, MAX_TRACKS_PER_SIGNAL) if b not in used)
            self.signals[signal_ID] = (base, NearestCenterTracker(), {})
            reset = list(range(base, base + MAX_TRACKS_PER_SIGNAL))
        else:
            reset = []
        base, tracker, slot_of = self.signals[signal_ID]
        n = len(cams)
        slots = np.full(n, -1, np.int32)
        if self.show_largest:
            slots[int(np.argmax(cams[:, 0]))] = base                               # main.py:129
            return slots, None, reset
        ids, fresh = tracker.update(np.asarray(cams)[:, [2, 1]] * 512.0)           # main.py:138
        for tid in list(slot_of):
            if tid not in tracker.tracks:
                del slot_of[tid]
        for i, tid in enumerate(ids):
            if tid not in slot_of:
                free = [s for s in range(base, base + MAX_TRACKS_PER_SIGNAL) if s not in slot_of.values()]
                if not free:
                    continue                                                       # more people than slots: left unsmoothed
                slot_of[tid] = free[0]
                reset.append(free[0])
            slots[i] = slot_of[tid]
        # two detections on one track in the same frame would race on the filter state: only the first keeps the slot
        seen = set()
        for i in range(n):
            if slots[i] >= 0:
                if slots[i] in seen:
                    slots[i] = -1
                seen.add(int(slots[i]))
        return slots, np.asarray(ids, np.int32), reset
