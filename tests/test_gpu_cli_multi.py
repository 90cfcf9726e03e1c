"""``--inputs`` on the GPU (romp_b200/cli.py ``run_inputs``): every input's output directory equals, file by file, what
``run_video`` of that input alone writes on a fresh instance (JPEG and PNG bytes, npz arrays bit for bit,
``video_results.npz``), for ROMP without -t, with -t and with -t --show_largest, and BEV without and with -t.

The inputs differ in size and length: three videos (one whose planted centres are empty, so nobody is detected), a
folder of frames of mixed sizes and, for BEV, a wide video that takes crowd mode.  People are planted through the
centre-map hook, which gives frame t of input i the map ``run_video``'s override gives it (row t % B of the input's
maps).  Each mode runs with --open_inputs below and above the number of inputs, and --max_batch below and above it.
The fixtures, and the release of every instance's conv graphs after each test, are those of tests/test_gpu_cli.py."""
import os
import subprocess
import sys
import types

import cv2
import numpy as np
import pytest
import torch

from romp_b200 import cli, synth
from romp_b200.bev import BEV, bev_settings
from romp_b200.main import ROMP, romp_settings
from tests.test_cli_multi_host import same_tree
from tests.test_gpu_cli import (ROOT, bev_files, frame_images, release_device_memory, romp_files,  # noqa: F401
                                write_folder)

pytestmark = pytest.mark.gpu

B = 8                                    # --max_batch of the single-input runs: rows of each input's planted maps
RUNS = [(2, 8), (8, 4)]                  # (--open_inputs, --max_batch): K below / above the inputs, max_batch above / below K


def write_video(path, n, h, w, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h, w, 3)).astype(np.int16)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 24, (w, h))
    assert vw.isOpened()
    for t in range(n):
        f = np.clip(base + rs.randint(-8, 9, base.shape), 0, 255).astype(np.uint8)
        f[h // 4:h // 2, (9 * t) % (w // 2):(9 * t) % (w // 2) + w // 5] = (30 * t) % 256
        vw.write(f)
    vw.release()
    return path


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """[(path, kind)]: kind "people", "empty" (planted maps all zero) or "wide" (BEV crowd mode, not planted)."""
    d = tmp_path_factory.mktemp("inputs")
    out = [(write_video(str(d / "walk.avi"), 29, 480, 640, 1), "people"),
           (write_video(str(d / "hall.avi"), 11, 720, 1280, 2), "people"),
           (write_folder(str(d / "mixed"), frame_images(19, seed=3)) and str(d / "mixed"), "people"),
           (write_video(str(d / "night.avi"), 7, 300, 580, 4), "empty")]
    wide = (write_video(str(d / "pano.avi"), 5, 360, 800, 5), "wide")
    return out, wide


def planted(model_kind, inputs_, seed):
    """Each input's planted centre maps, B rows (None for the wide input)."""
    maps = []
    for i, (_, kind) in enumerate(inputs_):
        if kind == "wide":
            maps.append(None)
            continue
        if model_kind == "romp":
            c, _ = synth.plant_centers(B, seed=seed + i)
        else:
            c, _ = synth.plant_centers_3d(B, seed=seed + i)
        if kind == "empty":
            c[:] = 0.0
        maps.append(torch.from_numpy(c).cuda())
    return maps


def hook_of(maps):
    return lambda i, t: None if maps[i] is None else maps[i][t % B]


def run_all(tmp_path, make, flags, inputs_, maps, prefix):
    """The single-input references, then --inputs at every (open_inputs, max_batch) of RUNS, compared file by file."""
    ref = str(tmp_path / "ref")
    for (p, _), co in zip(inputs_, maps):
        stem = os.path.splitext(os.path.basename(p))[0]
        args = types.SimpleNamespace(input=p, save_path=os.path.join(ref, stem), save_video=False, frame_rate=24)
        cli.run_video(make(flags + ["--max_batch", str(B)]), args, prefix, co)
    detected = 0
    for k, (open_inputs, max_batch) in enumerate(RUNS):
        extra = ["--open_inputs", str(open_inputs), "--max_batch", str(max_batch)]
        if "-t" in flags:
            extra += ["--video_streams", str(open_inputs)]
        model = make(flags + extra)
        out = str(tmp_path / f"out{k}")
        cli.run_inputs(model, [p for p, _ in inputs_], out, types.SimpleNamespace(open_inputs=open_inputs, save_video=False,
                                                                               frame_rate=24), prefix, hook_of(maps))
        same_tree(out, ref)
        for (p, kind) in inputs_:
            stem = os.path.splitext(os.path.basename(p))[0]
            npz = [n for n in os.listdir(os.path.join(out, stem)) if n.endswith(".npz") and n != "video_results.npz"]
            if kind == "empty":                                  # nobody: no npz, and no results in video_results.npz
                assert npz == []
                assert np.load(os.path.join(out, stem, "video_results.npz"), allow_pickle=True)["results"][()] == {}
            else:
                detected += len(npz)
    assert detected > 0
    return ref


@pytest.mark.parametrize("flags", [[], ["-t"], ["-t", "--show_largest"]], ids=["plain", "tracked", "largest"])
def test_romp_inputs_equal_single_input_runs(tmp_path, romp_files, inputs, flags):
    inputs_, _ = inputs
    base = ["--model_path", romp_files["model"], "--smpl_path", romp_files["smpl"]]
    make = lambda f: ROMP(romp_settings(base + f), state_dict=romp_files["sd"], smpl_pack=romp_files["pack"])
    ref = run_all(tmp_path, make, flags, inputs_, planted("romp", inputs_, 50), None)
    if flags == ["-t"]:
        res = np.load(os.path.join(ref, "walk", "video_results.npz"), allow_pickle=True)["sequence_results"][()]
        assert len(res) > 0                                      # tracks were followed across frames


@pytest.mark.parametrize("flags", [[], ["-t"]], ids=["plain", "tracked"])
def test_bev_inputs_equal_single_input_runs(tmp_path, bev_files, inputs, flags):
    inputs_, wide = inputs
    inputs_ = inputs_ + [wide]
    base = ["--model_path", bev_files["model"], "--smpl_path", bev_files["smpl"], "--smil_path", bev_files["smil_file"]]
    make = lambda f: BEV(bev_settings(base + f), state_dict=bev_files["sd"], smpla_pack=bev_files["smpla"],
                         smil_pack=bev_files["smil"])
    prefix = f"_2_{bev_settings([]).center_thresh}"
    ref = run_all(tmp_path, make, flags, inputs_, planted("bev", inputs_, 60), prefix)
    assert len(os.listdir(os.path.join(ref, "pano", "pano_frames"))) == 5


@pytest.mark.parametrize("module", ["romp.main", "bev.main"])
def test_python_m_inputs_with_save_video(tmp_path, romp_files, bev_files, inputs, module):
    inputs_, _ = inputs
    paths = [inputs_[0][0], inputs_[1][0]]             # one frame size each: the mp4 holds every frame
    out = str(tmp_path / "out")
    if module == "romp.main":
        flags = ["--model_path", romp_files["model"], "--smpl_path", romp_files["smpl"], "--max_batch", "8"]
    else:
        flags = ["--model_path", bev_files["model"], "--smpl_path", bev_files["smpl"], "--smil_path", bev_files["smil_file"],
                 "--max_batch", "8"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", module, "--mode", "video", "-t", "--inputs"] + paths +
                       ["-o", out, "--save_video", "--open_inputs", "2"] + flags,
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    assert sorted(os.listdir(out)) == ["hall", "walk"]
    for stem, n in (("walk", 29), ("hall", 11)):
        names = set(os.listdir(os.path.join(out, stem)))
        assert f"{stem}.mp4" in names and len([x for x in names if x.endswith(".png")]) == n
        cap = cv2.VideoCapture(os.path.join(out, stem, f"{stem}.mp4"))
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == n
        cap.release()
    assert len(os.listdir(os.path.join(out, "walk", "walk_frames"))) == 29
    if module == "romp.main":                                    # the calibrated head detects people
        assert os.path.exists(os.path.join(out, "walk", "video_results.npz"))
    bad = subprocess.run([sys.executable, "-m", module, "--mode", "video", "--inputs", paths[0], str(tmp_path / "nope"),
                          "-o", out] + flags, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert bad.returncode != 0 and "does not exist" in bad.stderr
