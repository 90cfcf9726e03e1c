"""CPU oracle of the temporal stage (row f4).  TEST INFRASTRUCTURE ONLY.

numpy (fp32) restatement of the reference's One-Euro smoothing: LowPassFilter (simple_romp/romp/utils.py:203-215),
OneEuroFilter (:217-246), create_OneEuroFilter (:258-259), smooth_results (:262-270), smooth_global_rot_matrix (:188-192)
with utils.batch_rodrigues / quat2mat (:493-533) and rotation_matrix_to_angle_axis (:535-552, via the quaternion code
:554-682 restated in oracle/romp_oracle.py).  Pinned by tests/test_oracle_golden.py::test_one_euro against
tests/golden/one_euro.npz (outputs of the reference's own functions; the --show_largest recurrence) and
::test_one_euro_tracked against tests/golden/one_euro_tracked.npz (the tracked recurrence, see smooth_tracked)."""
import numpy as np
import torch

from . import romp_oracle as R

F = np.float32


class OneEuro:
    def __init__(self, mincutoff, beta=0.7, dcutoff=1.0, freq=30.0):
        self.mincutoff, self.beta, self.dcutoff, self.freq = F(mincutoff), F(beta), F(dcutoff), F(freq)
        self.prev_raw = self.prev_x = self.prev_dx = None

    def alpha(self, cutoff):
        te = F(1.0) / self.freq
        tau = F(1.0) / (F(2 * np.pi) * cutoff)
        return F(1.0) / (F(1.0) + tau / te)

    def process(self, x):
        x = np.asarray(x, F)
        if self.prev_raw is None:
            edx = np.zeros_like(x)
            y = x
        else:
            dx = (x - self.prev_raw) * self.freq
            ad = self.alpha(self.dcutoff)
            edx = ad * dx + (F(1.0) - ad) * self.prev_dx
            a = self.alpha(self.mincutoff + self.beta * np.abs(edx))
            y = a * x + (F(1.0) - a) * self.prev_x
        self.prev_raw, self.prev_x, self.prev_dx = x, y.astype(F), edx.astype(F)
        return self.prev_x


def make_filters(smooth_coeff=3.0):
    return {"smpl_thetas": OneEuro(smooth_coeff), "cam": OneEuro(1.6), "smpl_betas": OneEuro(0.6), "global_rot": OneEuro(smooth_coeff)}


def rodrigues_quat(aa):
    """utils.batch_rodrigues (:493-505) + quat2mat (:507-533) for one axis-angle vector -> [9]."""
    aa = np.asarray(aa, F)
    nrm = np.sqrt(((aa + F(1e-8)) ** 2).sum(dtype=F), dtype=F)
    u = aa / nrm
    h = nrm * F(0.5)
    q = np.concatenate([[np.cos(h)], np.sin(h) * u]).astype(F)
    q = q / np.sqrt((q * q).sum(dtype=F), dtype=F)
    w, x, y, z = q
    return np.array([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z, 2 * w * z + 2 * x * y,
                     w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x, 2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z,
                     w * w - x * x - y * y + z * z], F)


def smooth(filters, thetas, betas, cam):
    """smooth_results (:262-270) for one person."""
    Rm = filters["global_rot"].process(rodrigues_quat(thetas[:3]))
    g = R.rotmat_to_aa(torch.from_numpy(Rm.reshape(1, 3, 3))).numpy().reshape(3)
    pose = filters["smpl_thetas"].process(thetas[3:])
    return np.concatenate([g, pose]).astype(F), filters["smpl_betas"].process(betas), filters["cam"].process(cam)


def smooth_tracked(filters, thetas, betas, cam):
    """One person of the tracked mode (romp/main.py:152-154, bev/main.py:283-285): thetas [72], betas, cam [3] are float32
    row VIEWS of the frame's outputs and receive the smoothed values in place.  OneEuro.process keeps the view it was
    given as prev_raw (np.asarray does not copy), as LowPassFilter keeps the tensor (utils.py:213), so the write-back
    turns prev_raw of body pose, betas and cam into the smoothed value and the next dx is taken against it; the
    global-rotation filter is fed a fresh matrix and keeps the raw one."""
    for v in (thetas, betas, cam):
        assert isinstance(v, np.ndarray) and v.dtype == F and v.base is not None, "smooth_tracked needs float32 row views"
    thetas[:], betas[:], cam[:] = smooth(filters, thetas, betas, cam)
