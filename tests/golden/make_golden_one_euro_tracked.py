"""Golden fixture for the TRACKED mode of the temporal path: the REFERENCE's create_OneEuroFilter / smooth_results
(simple_romp/romp/utils.py:188-270) driven exactly as ROMP.temporal_optimization drives them without --show_largest
(romp/main.py:148-154): every frame has new [n,72] / [n,10] / [n,3] tensors, smooth_results receives the row VIEWS
thetas[ind], betas[ind], cam[ind], and its three results are assigned back into those rows.  LowPassFilter keeps
prev_raw_value = value without a copy (utils.py:213), so from the second sample on the pose, betas and cam filters
differentiate against their previous SMOOTHED value; make_golden_one_euro.py is the --show_largest recurrence.

    python tests/golden/make_golden_one_euro_tracked.py          # build container only (needs /root/reference)

norfair (the reference's tracker) is not available, so the track ids are given: 6 persons over 48 frames in a different
row order every frame, person 3 absent in frames 10-14 (its filters resume from their old state), person 6 first seen in
frame 20, person 2's global rotation walking through pi.  Rows past n[t] are zero, ids -1.  The file is written with
fixed zip timestamps so that a rerun reproduces it byte for byte."""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import load_reference  # noqa: E402

T, P = 48, 6


def sequences():
    """-> per-person signals thetas [T,P,72], betas [T,P,10], cam [T,P,3] and the per-frame row order ids [T,P] (-1 pad)."""
    rs = np.random.RandomState(33)
    thetas = np.cumsum(rs.normal(0, 0.08, size=(T, P, 72)), 0).astype(np.float32) + rs.normal(0, 0.5, size=(1, P, 72)).astype(np.float32)
    axis = np.array([0.6, -0.64, 0.48])
    thetas[:, 1, :3] = (axis[None] * np.linspace(2.7, 3.6, T)[:, None] + rs.normal(0, 0.01, size=(T, 3))).astype(np.float32)
    betas = np.cumsum(rs.normal(0, 0.05, size=(T, P, 10)), 0).astype(np.float32)
    cam = (np.array([0.8, 0.0, 0.1], np.float32) + np.cumsum(rs.normal(0, 0.02, size=(T, P, 3)), 0)).astype(np.float32)
    ids = np.full((T, P), -1, np.int32)
    for t in range(T):
        present = [p + 1 for p in range(P) if not (p == 2 and 10 <= t <= 14) and not (p == 5 and t < 20)]
        ids[t, :len(present)] = rs.permutation(present)
    return thetas, betas, cam, ids


def save_npz_fixed(path, **arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for k, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(a), allow_pickle=False)
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(zi, buf.getvalue())


def main():
    U = load_reference()["romp.utils"]
    sig_t, sig_b, sig_c, ids = sequences()
    filters = {}
    n = (ids >= 0).sum(1).astype(np.int32)
    i_t, i_b, i_c = np.zeros_like(sig_t), np.zeros_like(sig_b), np.zeros_like(sig_c)
    o_t, o_b, o_c = np.zeros_like(sig_t), np.zeros_like(sig_b), np.zeros_like(sig_c)
    for t in range(T):
        rows = ids[t, :n[t]] - 1
        i_t[t, :n[t]], i_b[t, :n[t]], i_c[t, :n[t]] = sig_t[t, rows], sig_b[t, rows], sig_c[t, rows]
        outputs = {"smpl_thetas": torch.from_numpy(i_t[t, :n[t]].copy()), "smpl_betas": torch.from_numpy(i_b[t, :n[t]].copy()),
                   "cam": torch.from_numpy(i_c[t, :n[t]].copy())}
        for ind, tid in enumerate(ids[t, :n[t]].tolist()):                       # romp/main.py:148-154
            if tid not in filters:
                filters[tid] = U.create_OneEuroFilter(3.0)
            outputs["smpl_thetas"][ind], outputs["smpl_betas"][ind], outputs["cam"][ind] = \
                U.smooth_results(filters[tid], outputs["smpl_thetas"][ind], outputs["smpl_betas"][ind], outputs["cam"][ind])
        o_t[t, :n[t]], o_b[t, :n[t]], o_c[t, :n[t]] = outputs["smpl_thetas"].numpy(), outputs["smpl_betas"].numpy(), outputs["cam"].numpy()
    save_npz_fixed(os.path.join(HERE, "one_euro_tracked.npz"), thetas=i_t, betas=i_b, cam=i_c, ids=ids, n=n,
                   out_thetas=o_t, out_betas=o_b, out_cam=o_c)
    print("wrote one_euro_tracked.npz; max change by smoothing:", np.abs(o_t - i_t).max(), np.abs(o_c - i_c).max())


if __name__ == "__main__":
    main()
