"""Row f4 on the GPU: the One-Euro smoothing stage (csrc/temporal.cu) through the C ABI against the REFERENCE's own
smooth_results outputs (tests/golden/one_euro.npz), with interleaved slots and a slot reset; and ROMP.forward with
--temporal_optimize (both the --show_largest and the tracked mode) on a short synthetic sequence; the tracked mode against
the oracle's tracked recurrence (oracle/temporal_oracle.py::smooth_tracked) fed with the plain model's outputs and the
ids the run returned.  The kernel's two recurrences against float64: tests/test_gpu_romp_post_fp64.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from romp_b200 import ROMP, _lib, romp_settings, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def test_one_euro_kernel_matches_reference_sequences():
    z = np.load(os.path.join(HERE, "golden", "one_euro.npz"))
    T, P = z["thetas"].shape[:2]
    lib = _lib.load()
    h = lib.b200romp_tracks_create(0, 16)
    assert h
    slots = torch.tensor([5, 0, 9], dtype=torch.int32, device="cuda")          # persons use arbitrary, non-contiguous slots
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for rep in range(2):                                                       # second pass after a reset must repeat the first
        _lib.check(lib.b200romp_tracks_reset(h, -1, st))
        err = 0.0
        for t in range(T):
            th = torch.from_numpy(z["thetas"][t]).cuda().contiguous()
            be = torch.from_numpy(z["betas"][t]).cuda().contiguous()
            ca = torch.from_numpy(z["cam"][t]).cuda().contiguous()
            _lib.check(lib.b200romp_one_euro_smooth(h, C.c_void_p(slots.data_ptr()), P, None, C.c_void_p(th.data_ptr()),
                                                    C.c_void_p(be.data_ptr()), 10, 10, C.c_void_p(ca.data_ptr()), 3.0, 30.0, 0, st))
            torch.cuda.synchronize()
            err = max(err, np.abs(th.cpu().numpy() - z["out_thetas"][t]).max(), np.abs(be.cpu().numpy() - z["out_betas"][t]).max(),
                      np.abs(ca.cpu().numpy() - z["out_cam"][t]).max())
        print(f"pass {rep}: max |kernel - reference| over {T} frames x {P} persons = {err:.2e}")
        assert err < 3e-5
    lib.b200romp_tracks_destroy(h)


@pytest.mark.parametrize("largest", [False, True])
def test_forward_with_temporal_optimize(largest):
    from oracle import romp_oracle as O
    from oracle import temporal_oracle as T
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    rs = np.random.RandomState(7)
    base = rs.randint(0, 256, (512, 512, 3)).astype(np.uint8)
    c, _ = O.romp_maps(sd, np.ascontiguousarray(base[None, :, :, ::-1]))
    sd2, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    flags = ["--precision", "fp32", "--max_batch", "1", "-t"] + (["--show_largest"] if largest else [])
    m = ROMP(romp_settings(flags), state_dict=sd2, smpl_pack=pack)
    plain = ROMP(romp_settings(["--precision", "fp32", "--max_batch", "1"]), state_dict=sd2, smpl_pack=pack)
    outs, filters = [], {}
    for t in range(6):
        img = np.clip(base.astype(np.int32) + rs.randint(-6, 7, base.shape), 0, 255).astype(np.uint8)   # small frame-to-frame change
        o, p = m(img), plain(img)
        assert o is not None and p is not None
        n = len(p["cam"])
        assert o["center_preds"].shape[0] == n and o["global_orient"].shape == (n, 3)
        if largest:
            assert o["smpl_thetas"].shape == (1, 72) and o["verts"].shape == (1, 6890, 3) and "track_ids" not in o
        else:
            assert o["smpl_thetas"].shape == (n, 72) and o["track_ids"].shape == (n,) and o["track_ids"].dtype == np.int32
        if t == 0:       # the first sample passes through the filters unchanged (rotation: matrix round trip)
            k = int(np.argmax(p["cam"][:, 0])) if largest else slice(None)
            assert np.abs(o["cam"] - p["cam"][k]).max() < 1e-6 and np.abs(o["smpl_thetas"][..., 3:] - p["smpl_thetas"][k][..., 3:]).max() < 1e-6
            assert np.abs(o["smpl_thetas"][..., :3] - p["smpl_thetas"][k][..., :3]).max() < 1e-4
        if not largest:  # every frame equals the reference's tracked recurrence on the unsmoothed outputs (departs at frame 2 otherwise)
            th, be, ca = p["smpl_thetas"].copy(), p["smpl_betas"].copy(), p["cam"].copy()
            first = {int(tid): r for r, tid in reversed(list(enumerate(o["track_ids"])))}
            for tid, r in first.items():     # a second detection on one track in a frame is left unsmoothed (temporal.py)
                T.smooth_tracked(filters.setdefault(tid, T.make_filters(3.0)), th[r], be[r], ca[r])
            assert np.abs(o["smpl_thetas"][:, 3:] - th[:, 3:]).max() < 3e-5, t
            assert np.abs(o["smpl_betas"] - be).max() < 3e-5 and np.abs(o["cam"] - ca).max() < 3e-5, t
        # SMPL ran on the smoothed parameters
        v, j = O.smpl_forward(pack, o["smpl_betas"], o["smpl_thetas"])
        assert np.abs(o["verts"] - v.numpy()).max() < 1e-4
        outs.append(o)
    if not largest:
        assert np.array_equal(outs[0]["track_ids"], outs[1]["track_ids"])       # same people, same ids
    assert np.abs(outs[2]["cam"] - outs[1]["cam"]).max() > 0                   # and the filter state moves
