"""Stream mode (--video_streams) without a GPU: the settings checks, the host's stream-index bookkeeping, the declared
and bound C ABI, and the track kernels' registers and shared memory (compiled for sm_90a here)."""
import os
import re
import subprocess
import tempfile
from types import SimpleNamespace

import pytest

from romp_b200 import _lib
from romp_b200.bev import bev_settings
from romp_b200.main import romp_settings
from romp_b200.streams import MAX_VIDEO_STREAMS, check_video_streams, stream_indices

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_settings_default_and_checks():
    assert romp_settings([]).video_streams == 0 and bev_settings([]).video_streams == 0
    assert check_video_streams(romp_settings(["-t", "--video_streams", "8"]), True) == 8
    assert check_video_streams(bev_settings(["--video_streams", str(MAX_VIDEO_STREAMS)]), True) == MAX_VIDEO_STREAMS
    assert check_video_streams(SimpleNamespace(), False) == 0
    for n, temporal in ((3, False), (MAX_VIDEO_STREAMS + 1, True), (-1, True)):
        with pytest.raises(ValueError):
            check_video_streams(SimpleNamespace(video_streams=n), temporal)


def test_stream_indices_take_free_indices_and_refuse_overflow():
    live, resets = {}, []
    assert stream_indices(live, ["a", "b", "a", 7], 3, resets.append) == [0, 1, 0, 2]
    assert resets == [0, 1, 2]
    with pytest.raises(ValueError):                  # a 4th live stream: refused before any reset
        stream_indices(live, ["a", "c"], 3, resets.append)
    assert resets == [0, 1, 2] and set(live) == {"a", "b", 7}
    live.pop("b")                                    # reset_temporal("b")
    assert stream_indices(live, ["c", 7, "b"][:2], 3, resets.append) == [1, 2]
    assert resets == [0, 1, 2, 1]                    # "c" took b's index, which was reset first


def test_stream_symbols_declared_and_bound():
    text = open(os.path.join(ROOT, "include", "b200romp.h")).read()
    for sym in ("b200romp_bev_tracker_create_streams", "b200romp_romp_tracker_create_streams", "b200romp_romp_tracker_reset_stream"):
        assert re.search(r"\b%s\s*\(" % sym, text) and sym in _lib.EXPORTS
        assert "_sig(lib.%s," % sym in open(os.path.join(ROOT, "romp_b200", "_lib.py")).read()
    assert "#define B200ROMP_MAX_VIDEO_STREAMS %d" % MAX_VIDEO_STREAMS in text


def test_track_kernels_do_not_spill_and_smem_is_documented():
    nvcc = _lib._nvcc()
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    kernels = {}
    with tempfile.TemporaryDirectory() as tmp:
        for src in ("track.cu", "romp_track.cu"):
            r = subprocess.run([nvcc, "-c"] + _lib.NVCC_FLAGS + ["-Xptxas", "-v", "-o", os.path.join(tmp, "k.o"),
                                                                os.path.join(_lib.CSRC, src)], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            for name, spill in re.findall(r"Function properties for _ZN8b200romp\d+([a-z_]+_kernel)\w*\n\s*\d+ bytes stack frame, (\d+) bytes spill",
                                          r.stderr):
                kernels[name] = int(spill)
        probe = os.path.join(tmp, "probe.cu")
        with open(probe, "w") as f:
            f.write('#include <cstdio>\n#include "%s"\n#include "%s"\nnamespace b200romp { void set_error(const char*, ...) {} }\n'
                    'int main() { printf("%%zu %%zu\\n", b200romp::kTrkSmem, b200romp::kRtSmem); }\n'
                    % (os.path.join(_lib.CSRC, "track.cu"), os.path.join(_lib.CSRC, "romp_track.cu")))
        exe = os.path.join(tmp, "probe")
        r = subprocess.run([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, probe],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        trk, rt = map(int, subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split())
    assert {"bev_track_streams_kernel", "romp_track_streams_kernel", "bev_track_compact_kernel"} <= set(kernels)
    assert all(v == 0 for v in kernels.values()), kernels
    text = open(os.path.join(ROOT, "include", "b200romp.h")).read()
    assert "CTA: {:,} bytes".format(trk) in text.replace("\n * ", " ") and "CTA: {:,} bytes".format(rt) in text.replace("\n * ", " ")
    assert 2 * trk <= 227 * 1024                     # two BEV streams per SM
