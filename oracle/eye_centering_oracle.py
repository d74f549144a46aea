"""TEST INFRASTRUCTURE ONLY: float64 restatement of the reference's ``position_to_given_location``
(my_utils/eye_centering.py:35-66), pinned against the *unmodified* reference function by oracle/make_sampler_golden.py.

The reference solves ``d = (s, s bx, s by) M`` with ``M = [[e1x e2x e1y e2y], [1 1 0 0], [0 0 1 1]]`` by ``d pinv(M)``, the
minimum-norm least-squares solution; M has full row rank whenever the eyes differ in x or y, and then the normal
equations give the closed form below.  Plain numpy / torch, CPU; only tests/ and the golden script import this module."""
import numpy as np

EYE_VERTICES = (4051, 4597)
EYE_TARGETS = np.float32([-0.2419, 0.2441, 0.0501 - 0.1, 0.0509 - 0.1]).astype(np.float64)   # x1, x2, y1, y2


def eye_camera(eye1, eye2, targets=EYE_TARGETS):
    """eye1, eye2 (B, >=2) the two eye vertices -> cam (B, 3) float64 = (-s, bx, by).  Same operation order as
    gifb200_eye_camera, so the kernel's float32 result is this value rounded once."""
    e1x, e1y = np.asarray(eye1[:, 0], np.float64), np.asarray(eye1[:, 1], np.float64)
    e2x, e2y = np.asarray(eye2[:, 0], np.float64), np.asarray(eye2[:, 1], np.float64)
    x1, x2, y1, y2 = (float(t) for t in targets)
    dex, dey = e1x - e2x, e1y - e2y
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (dex * (x1 - x2) + dey * (y1 - y2)) / (dex * dex + dey * dey)
        sbx = 0.5 * (x1 + x2) - s * (0.5 * (e1x + e2x))
        sby = 0.5 * (y1 + y2) - s * (0.5 * (e1y + e2y))
        return np.stack([-s, sbx / s, sby / s], 1)


def projected_eyes(eye1, eye2, cam):
    """The eye positions in the normalised image under ``cam``, in the convention of the reference's
    tests/test_eye_positioning.py:63-72: (e[:2] + cam[1:]) * cam[0], y negated.  -> (B, 2, 2) float64 [eye1, eye2]."""
    cam = np.asarray(cam, np.float64)
    out = []
    for e in (eye1, eye2):
        p = (np.asarray(e[:, :2], np.float64) + cam[:, 1:3]) * cam[:, 0:1]
        p[:, 1] *= -1
        out.append(p)
    return np.stack(out, 1)
