"""The ``romp`` and ``bev`` command lines on the GPU (romp_b200/cli.py): video mode through the batched entry points,
saved file by file, against the per-frame calls the reference's loop makes, array for array and bit for bit.

Synthetic weights (romp_b200.synth) are written to temporary .pth files so that ``main()`` runs unchanged; ROMP's centre
head is calibrated to detect people, and people are planted through ``cli.run_frames``' centre-map override where frames
without anybody are needed.  70 frames at --max_batch 32 make three lists, the last one partial."""
import gc
import os
import subprocess
import sys

import cv2
import numpy as np
import pytest
import torch

from romp_b200 import cli, graph, synth
from romp_b200.bev import BEV, bev_settings
from romp_b200.bev import main as bev_main
from romp_b200.bev import run_image
from romp_b200.main import ROMP, img_preprocess, romp_settings
from romp_b200.main import main as romp_main

pytestmark = pytest.mark.gpu


_MODELS = []


@pytest.fixture(autouse=True)
def release_device_memory(monkeypatch):
    """Each test builds several full-size ROMP / BEV instances, main() included.  Their conv graphs live in the library
    (cudaMalloc'd weights and workspaces) until ``b200romp_net_destroy``, which the instances do not call, so every
    instance a test builds is recorded here and its graphs destroyed after the test; then the instances are collected
    (a ROMP instance only by the cycle collector: its ``model`` refers back to it) and PyTorch's cached blocks handed
    back to the driver.  The suites after this one find the device as free as before it."""
    for cls in (ROMP, BEV):
        def init(self, *a, _init=cls.__init__, **k):
            _init(self, *a, **k)
            _MODELS.append(self)
        monkeypatch.setattr(cls, "__init__", init)
    yield
    torch.cuda.synchronize()
    for m in _MODELS:
        for nets in m._nets.values():
            for g in nets:
                if isinstance(g, graph.NetBuilder):
                    m.lib.b200romp_net_destroy(g.net)
        m._nets.clear()
    _MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, B = 70, 32
SIZES = [(480, 640), (720, 1280), (512, 512), (1280, 720), (300, 580)]


def frame_images(n, seed):
    """Mixed content and sizes: noise, a noisy scene with a moving block, flat frames."""
    rs = np.random.RandomState(seed)
    out = []
    for t in range(n):
        h, w = SIZES[t % len(SIZES)]
        kind = t % 4
        if kind == 3:
            img = np.full((h, w, 3), (37 * t) % 256, np.uint8)
        else:
            img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
            if kind == 1:
                img[h // 4:h // 2, (5 * t) % (w // 2):(5 * t) % (w // 2) + w // 4] = 200
        out.append(img)
    return out


def write_folder(folder, images):
    os.makedirs(folder)
    for t, img in enumerate(images):
        assert cv2.imwrite(os.path.join(folder, f"f{t:04d}.png"), img)
    return [os.path.join(folder, f"f{t:04d}.png") for t in range(len(images))]


def save_pth(obj, path):
    torch.save({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in obj.items()}, path)
    return path


@pytest.fixture(scope="module")
def romp_files(tmp_path_factory):
    from oracle import romp_oracle as O
    d = tmp_path_factory.mktemp("romp_weights")
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    c, _ = O.romp_maps(sd, np.concatenate([img_preprocess(x)[0] for x in frame_images(2, seed=9)]))
    sd, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    return dict(sd=sd, pack=pack, model=save_pth(sd, str(d / "ROMP.pkl")), smpl=save_pth(pack, str(d / "SMPL_NEUTRAL.pth")))


@pytest.fixture(scope="module")
def bev_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("bev_weights")
    sd, smpla, smil = synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)
    return dict(sd=sd, smpla=smpla, smil=smil, model=save_pth(sd, str(d / "BEV.pth")), smpl=save_pth(smpla, str(d / "SMPLA.pth")),
                smil_file=save_pth(smil, str(d / "smil.pth")))


@pytest.fixture(scope="module")
def video_folder(tmp_path_factory):
    images = frame_images(N, seed=11)
    return write_folder(str(tmp_path_factory.mktemp("frames") / "clip"), images)


def romp_flags(files):
    return ["--model_path", files["model"], "--smpl_path", files["smpl"], "--max_batch", str(B)]


def bev_flags(files):
    return ["--model_path", files["model"], "--smpl_path", files["smpl"], "--smil_path", files["smil_file"], "--max_batch", str(B)]


def same(a, b, what):
    assert (a is None) == (b is None), what
    if a is None:
        return
    assert sorted(a) == sorted(b), (what, sorted(a), sorted(b))
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), (what, k)


def saved(out_dir, frame_path, prefix=""):
    """(result dict or None, PNG pixels) of one frame's files."""
    stem = os.path.join(out_dir, os.path.splitext(os.path.basename(frame_path))[0] + prefix)
    assert os.path.exists(stem + ".png"), stem
    npz = stem + ".npz"
    return (np.load(npz, allow_pickle=True)["results"][()] if os.path.exists(npz) else None), cv2.imread(stem + ".png")


def check_files(out_dir, paths, expected, prefix=""):
    """Every frame: its npz equals the expected result (no npz where None), its PNG is the input frame; and
    video_results.npz equals one built from the expected results."""
    for t, (p, exp) in enumerate(zip(paths, expected)):
        got, png = saved(out_dir, p, prefix)
        same(got, exp, f"frame {t}")
        assert np.array_equal(png, cv2.imread(p)), t
    ref_dir = out_dir + "_expected"
    s = cli.ResultSaver("video", ref_dir)
    for p, exp in zip(paths, expected):
        s(None if exp is None else dict(exp), p, prefix[1:] if prefix else None)
    cli.save_video_results(s.frame_save_paths)
    got = np.load(os.path.join(out_dir, "video_results.npz"), allow_pickle=True)
    exp = np.load(os.path.join(ref_dir, "video_results.npz"), allow_pickle=True)
    g, e = got["results"][()], exp["results"][()]
    assert list(g) == list(e)
    for k in g:
        same(g[k], e[k], k)
    gs, es = got["sequence_results"][()], exp["sequence_results"][()]
    assert list(gs) == list(es)
    for tid in gs:
        assert list(gs[tid]) == list(es[tid]) and gs[tid]["frame_id"] == es[tid]["frame_id"]
        for k in gs[tid]:
            assert len(gs[tid][k]) == len(es[tid][k])
            for x, y in zip(gs[tid][k], es[tid][k]):
                assert np.array_equal(np.asarray(x), np.asarray(y)), (tid, k)


ROMP_MODES = [[], ["-t"], ["-t", "--show_largest"]]


@pytest.mark.parametrize("flags", ROMP_MODES, ids=["plain", "tracked", "largest"])
def test_romp_video_main_equals_per_frame_forward(tmp_path, romp_files, video_folder, flags):
    """``romp --mode video`` through main(): each frame's npz is ``model(image)`` on a fresh instance."""
    out = str(tmp_path / "out")
    romp_main(["--mode", "video", "-i", os.path.dirname(video_folder[0]), "-o", out] + romp_flags(romp_files) + flags)
    make = lambda: ROMP(romp_settings(romp_flags(romp_files) + flags), state_dict=romp_files["sd"], smpl_pack=romp_files["pack"])
    ref = make()
    loop = [ref(cv2.imread(p)) for p in video_folder]
    assert sum(e is not None for e in loop) > N // 2
    if not flags:
        check_files(out, video_folder, loop)
        return
    # -t: forward_video is bit-identical however a video is cut into lists, so one frame per call on a fresh instance
    # is the exact reference; forward() per frame agrees within the tolerances of tests/test_gpu_romp_video.py
    one = make()
    exact = [one.forward_video([cv2.imread(p)])[0] for p in video_folder]
    check_files(out, video_folder, exact)
    tol = dict(smpl_thetas=1e-6, smpl_betas=1e-6, cam=1e-6, cam_trans=1e-6, global_orient=1e-6, body_pose=1e-6,
               center_confs=1e-6, verts=1e-5, joints=1e-5, pj2d_org=1e-3)
    for t, (a, b) in enumerate(zip(exact, loop)):
        assert (a is None) == (b is None) and (a is None or sorted(a) == sorted(b)), t
        for k in ([] if a is None else a):
            assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype, (t, k)
            if k in ("track_ids", "center_preds"):
                assert np.array_equal(a[k], b[k]), (t, k)
            elif a[k].size:
                assert float(np.abs(a[k].astype(np.float64) - b[k]).max()) <= tol[k], (t, k)
    if flags == ["-t"]:
        assert any("track_ids" in e for e in exact if e is not None)


def planted_romp(seed, empty):
    c, _ = synth.plant_centers(B, seed=seed)
    c[list(empty)] = 0.0
    return torch.from_numpy(c).cuda()


@pytest.mark.parametrize("flags", ROMP_MODES, ids=["plain", "tracked", "largest"])
def test_romp_video_frames_without_people(tmp_path, romp_files, video_folder, flags):
    """Planted centres with empty rows: those frames get a PNG and no npz; the others equal the per-frame call with the
    same centres (forward_images / forward_video of one frame, which forward() is, on a fresh instance)."""
    co = planted_romp(seed=21, empty=(3, 17))
    make = lambda: ROMP(romp_settings(romp_flags(romp_files) + flags), state_dict=romp_files["sd"], smpl_pack=romp_files["pack"])
    out = str(tmp_path / "out")
    frames, _ = cli.frame_source(os.path.dirname(video_folder[0]), out)
    cli.run_frames(make(), frames, cli.ResultSaver("video", out, writers=cli.WRITERS), None, co)
    ref = make()
    one = (lambda img, c: ref.forward_video([img], center_override=c)[0]) if flags else \
        (lambda img, c: ref.forward_images([img], center_override=c)[0])
    expected = [one(cv2.imread(p), co[t % B:t % B + 1]) for t, p in enumerate(video_folder)]
    empty = [t for t in range(N) if t % B in (3, 17)]
    assert all(expected[t] is None for t in empty) and sum(e is not None for e in expected) == N - len(empty)
    for t in empty:
        assert not os.path.exists(os.path.join(out, f"f{t:04d}.npz")) and os.path.exists(os.path.join(out, f"f{t:04d}.png"))
    cli.save_video_results([os.path.join(out, f"f{t:04d}.png") for t in range(N)])
    check_files(out, video_folder, expected)


def planted_bev(seed, empty):
    vol, _ = synth.plant_centers_3d(B, seed=seed)
    vol[list(empty)] = 0.0
    return torch.from_numpy(vol).cuda()


@pytest.fixture(scope="module")
def bev_video(tmp_path_factory):
    """The 70 frames with two 1080x3840 crowd-mode frames in the middle."""
    images = frame_images(N, seed=11)
    rs = np.random.RandomState(12)
    for k in (0, 1):
        images.insert(N // 2 + k, rs.randint(0, 256, (1080, 3840, 3)).astype(np.uint8))
    return write_folder(str(tmp_path_factory.mktemp("bev_frames") / "clip"), images)


def normal_index(paths):
    """For every frame: its index among the normal (not wide) frames of its list of B, or None for a wide frame."""
    out = []
    for l0 in range(0, len(paths), B):
        k = 0
        for p in paths[l0:l0 + B]:
            h, w = cv2.imread(p).shape[:2]
            out.append(None if w / h >= 2 else k)
            k += w / h < 2
    return out


@pytest.mark.parametrize("flags", [[], ["-t"]], ids=["plain", "tracked"])
def test_bev_video_equals_forward_images(tmp_path, bev_files, bev_video, flags):
    co = planted_bev(seed=31, empty=(4,))
    make = lambda: BEV(bev_settings(bev_flags(bev_files) + flags), state_dict=bev_files["sd"], smpla_pack=bev_files["smpla"],
                       smil_pack=bev_files["smil"])
    s = bev_settings(bev_flags(bev_files))
    prefix = f"_2_{s.center_thresh}"
    out = str(tmp_path / "out")
    frames, _ = cli.frame_source(os.path.dirname(bev_video[0]), out)
    cli.run_frames(make(), frames, cli.ResultSaver("video", out, writers=cli.WRITERS), prefix, co)
    cli.save_video_results([os.path.join(out, os.path.splitext(os.path.basename(p))[0] + f"_{prefix}.png") for p in bev_video])
    imgs = [cv2.imread(p) for p in bev_video]
    kidx = normal_index(bev_video)
    ref = make()
    if flags:
        normal = [t for t, k in enumerate(kidx) if k is not None]
        co_all = torch.cat([co[kidx[t]:kidx[t] + 1] for t in normal])
        expected = ref.forward_images(imgs, center3d_override=co_all)
    else:
        expected = [ref.forward_images([img], center3d_override=co[k:k + 1])[0] if k is not None else None
                    for img, k in zip(imgs, kidx)]
    wide_ref = make()
    for t, k in enumerate(kidx):
        if k is None:
            long = wide_ref.process_long_image(imgs[t])
            if flags:
                same(expected[t], long, f"wide frame {t}")
            expected[t] = long
    assert sum(k is None for k in kidx) == 2
    if not flags:
        assert all(expected[t] is None for t, k in enumerate(kidx) if k == 4)
    assert sum(e is not None for e in expected) > N // 2
    check_files(out, bev_video, expected, "_" + prefix)
    if flags:
        assert any("track_ids" in e for e in expected if e is not None)


def test_bev_image_mode(tmp_path, bev_files, bev_video):
    """``bev --mode image``: ResultSaver('image') names with the prefix {center_thresh}; the normal image equals
    forward_images with the same planted centres, the wide one process_long_image."""
    co = planted_bev(seed=32, empty=())
    s = bev_settings(bev_flags(bev_files))
    make = lambda: BEV(s, state_dict=bev_files["sd"], smpla_pack=bev_files["smpla"], smil_pack=bev_files["smil"])
    model, ref = make(), make()
    normal, wide = bev_video[1], bev_video[N // 2]
    run_image(model, normal, str(tmp_path / "res.jpg"), s.center_thresh, co[:1])
    got = np.load(str(tmp_path / f"res_{s.center_thresh}.npz"), allow_pickle=True)["results"][()]
    same(got, ref.forward_images([cv2.imread(normal)], center3d_override=co[:1])[0], "normal image")
    assert cv2.imread(str(tmp_path / f"res_{s.center_thresh}.jpg")).shape == cv2.imread(normal).shape
    run_image(model, wide, str(tmp_path / "dir"), s.center_thresh)
    stem = os.path.splitext(os.path.basename(wide))[0]
    exp = ref.process_long_image(cv2.imread(wide))
    got, png = saved(str(tmp_path / "dir"), wide, f"_{s.center_thresh}")
    same(got, exp, "wide image")
    assert np.array_equal(png, cv2.imread(wide))
    names = sorted(os.listdir(str(tmp_path / "dir")))
    assert names == sorted([f"{stem}_{s.center_thresh}.png"] + ([f"{stem}_{s.center_thresh}.npz"] if exp is not None else []))
    # main() on the same image: the file set of a directory save path
    bev_main(["-i", normal, "-o", str(tmp_path / "main")] + bev_flags(bev_files))
    assert os.path.exists(str(tmp_path / "main" / f"{os.path.splitext(os.path.basename(normal))[0]}_{s.center_thresh}.png"))


@pytest.mark.parametrize("module", ["romp.main", "bev.main"])
def test_python_m_video_with_save_video(tmp_path, romp_files, bev_files, module):
    rs = np.random.RandomState(41)                # one frame size, as in a video: the mp4 holds frames of the first's size
    images = [rs.randint(0, 256, (480, 640, 3)).astype(np.uint8) for _ in range(12)]
    folder = str(tmp_path / "clip")
    paths = write_folder(folder, images)
    out = str(tmp_path / "out")
    flags = romp_flags(romp_files) if module == "romp.main" else bev_flags(bev_files)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", module, "--mode", "video", "-i", folder, "-o", out, "--save_video"] + flags,
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    prefix = "" if module == "romp.main" else f"__2_{bev_settings([]).center_thresh}"
    stems = [os.path.splitext(os.path.basename(p))[0] + prefix for p in paths]
    names = set(os.listdir(out))
    assert {s + ".png" for s in stems} <= names and "video_results.npz" in names and "clip.mp4" in names
    npz = {n for n in names if n.endswith(".npz")} - {"video_results.npz"}
    assert npz <= {s + ".npz" for s in stems}
    assert names == {s + ".png" for s in stems} | npz | {"video_results.npz", "clip.mp4"}
    res = np.load(os.path.join(out, "video_results.npz"), allow_pickle=True)["results"][()]
    assert set(res) == {n[:-4] + ".png" for n in npz}
    if module == "romp.main":
        assert len(npz) == 12                                       # the calibrated head detects in every frame
    cap = cv2.VideoCapture(os.path.join(out, "clip.mp4"))
    assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 12
    cap.release()
