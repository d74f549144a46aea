"""CPU: the float64 eye-centring restatement against the unmodified reference's position_to_given_location
(tests/golden/eye_centering.npz, oracle/make_sampler_golden.py), the seeded parameter draw of tools/sample_faces.py, and the
C entry points of the sampler's two kernels reporting shape errors through return codes."""
import os
import re
import sys

import numpy as np

import golden_util as gu
from oracle import eye_centering_oracle as EO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def recorded_pinv_bar():
    """Per camera column, max|float64 restatement - reference float32 pinverse| as the golden's note records it."""
    txt = open(os.path.join(gu.GOLDEN_DIR, "EYE_CENTERING_ORACLE_VS_REFERENCE.txt")).read()
    return np.array([float(re.search(rf"cam\[{c}\] max\|oracle\(f32 verts\) - reference\| = (\S+)", txt).group(1))
                     for c in ("scale", "tx", "ty")])


def test_restatement_matches_reference_golden():
    g = gu.load_golden("eye_centering.npz")
    cam = EO.eye_camera(g["eyes"][:, 0], g["eyes"][:, 1])
    bar = recorded_pinv_bar()
    np.testing.assert_allclose(bar, g["pinv_err"], rtol=1e-3)
    err = np.abs(cam - g["cam_ref"].astype(np.float64)).max(0)
    assert (err <= bar * (1 + 1e-3)).all(), (err, bar)
    # the bar is float32 rounding of the pseudo-inverse, not a disagreement: about one part in a million of the scale
    # (|scale| 7..9) and well under a micro-unit of translation (the head spans ~0.2 units)
    assert bar[0] <= 64 * np.finfo(np.float32).eps * np.abs(g["cam_ref"][:, 0]).max() and (bar[1:] < 2e-6).all(), bar
    assert tuple(g["eye_vertices"]) == EO.EYE_VERTICES and np.array_equal(g["targets"], EO.EYE_TARGETS.astype(np.float32))


def test_closed_form_is_the_pseudo_inverse_solution():
    """The closed form equals d . pinv(M) (the reference's formula) evaluated in float64."""
    g = gu.load_golden("eye_centering.npz")
    e1, e2 = g["eyes_f64"][:, 0], g["eyes_f64"][:, 1]
    cam = EO.eye_camera(e1, e2)
    for i in range(e1.shape[0]):
        M = np.array([[e1[i, 0], e2[i, 0], e1[i, 1], e2[i, 1]], [1, 1, 0, 0], [0, 0, 1, 1]], np.float64)
        s, sbx, sby = EO.EYE_TARGETS @ np.linalg.pinv(M)
        np.testing.assert_allclose(cam[i], [-s, sbx / s, sby / s], rtol=1e-11, atol=1e-13)
    # the fitted camera places the eyes' midpoint exactly (the residuals of the two eyes cancel)
    mid = EO.projected_eyes(e1, e2, cam).mean(1)
    x1, x2, y1, y2 = EO.EYE_TARGETS
    np.testing.assert_allclose(mid, np.broadcast_to([-(x1 + x2) / 2, (y1 + y2) / 2], mid.shape), atol=1e-13)
    # coincident eyes: no unique camera, NaN rather than an exception
    assert np.isnan(EO.eye_camera(e1[:1], e1[:1])).all()


def test_sample_faces_parameter_draw():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sample_faces as SF
    from gif_b200.conditions import DECA_COLUMNS, DECA_SLICES
    from gif_b200.flame_synth import synthetic_deca_params
    a, b, c = SF.draw_rows(40, 3), SF.draw_rows(40, 3), SF.draw_rows(40, 4)
    assert a.shape == (40, DECA_COLUMNS) and a.dtype == np.float32
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    col = lambda k: a[:, slice(*DECA_SLICES[k])]
    for k in ("shape", "exp"):
        assert (col(k)[:, 3:] == 0).all() and (col(k)[:, :3] != 0).all()
    pose = col("pose")
    assert (pose[:, [0, 2, 4, 5]] == 0).all()
    assert (np.abs(pose[:, 1]) <= np.pi / 8).all() and ((pose[:, 3] >= 0) & (pose[:, 3] <= np.pi / 12)).all()
    assert (col("tex") != 0).all()
    src = synthetic_deca_params(40, 3).numpy()
    for k in ("cam", "lit"):
        assert np.array_equal(col(k), src[:, slice(*DECA_SLICES[k])])
    given = synthetic_deca_params(3, 9).numpy()
    d = SF.draw_rows(7, 3, given)
    assert np.array_equal(d[:, 156:159], given[np.arange(7) % 3, 156:159]) and np.array_equal(d[:, 209:236], given[np.arange(7) % 3, 209:236])
    ids = SF.draw_identities(40, 100, 3)
    assert np.array_equal(ids, SF.draw_identities(40, 100, 3)) and ids.min() >= 0 and ids.max() < 100
    p = SF.params_to_save(a, ids)
    assert sorted(p) == sorted(["cam", "shape", "exp", "pose", "light_code", "texture_code", "identity_indices"])
    assert p["light_code"].shape == (40, 9, 3) and p["shape"].shape == (40, 100) and p["texture_code"].shape == (40, 50)


def test_kernel_entry_points_report_shape_errors():
    from gif_b200 import _lib
    lib = _lib.lib
    rc = lib.gifb200_eye_camera(None, None, 4, 5023, 4051, 5023, 0.0, 0.0, 0.0, 0.0, None)
    assert rc == -1 and b"eye vertex index" in lib.gifb200_last_error()
    rc = lib.gifb200_eye_camera(None, None, 4, 5023, -1, 4597, 0.0, 0.0, 0.0, 0.0, None)
    assert rc == -1 and b"eye vertex index" in lib.gifb200_last_error()
    assert lib.gifb200_eye_camera(None, None, 0, 5023, 4051, 4597, 0.0, 0.0, 0.0, 0.0, None) == 0     # empty batch: no launch
    rc = lib.gifb200_image_to_u8(None, None, 0, 8, 8, 192, 64, 8, 1, None)
    assert rc == -1 and b"image_to_u8" in lib.gifb200_last_error()
