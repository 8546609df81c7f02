"""CPU checks of tests/opq_reference.py: the v5 split and the rotation it reproduces (no GPU)."""
import numpy as np

from tests import ivf_reference as R
from tests import opq_reference as O


def _header(version, d, reserved0):
    h = np.zeros(1, R.HEADER)
    h["magic"], h["version"], h["d"], h["reserved0"] = b"B2IX", version, d, reserved0
    return h.tobytes()


def test_split_v5_strips_the_rotation_and_restores_the_version():
    d = 6
    rot = np.linalg.qr(np.random.default_rng(1).standard_normal((d, d)))[0].astype(np.float32)
    body = b"\x07" * 40
    for reserved0, want in ((0, 2), (4, 3)):
        got, r = O.split_v5(_header(5, d, reserved0) + body + rot.tobytes())
        h = np.frombuffer(got, R.HEADER, count=1)[0]
        assert h["version"] == want and h["reserved0"] == reserved0 and got[R.HEADER.itemsize:] == body
        assert r.tobytes() == rot.tobytes()
        assert O.orthonormal_error(r) < 1e-6


def test_rotate_f32_is_the_fmaf_chain_and_close_to_float64():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((5, 24)).astype(np.float32)
    rot = np.linalg.qr(rng.standard_normal((24, 24)))[0].astype(np.float32)
    y = O.rotate_f32(x, rot)
    want = np.zeros((5, 24), np.float32)
    for j in range(24):
        for r in range(5):
            acc = np.float32(0)
            for i in range(24):
                acc = np.float32(np.float64(acc) + np.float64(x[r, i]) * np.float64(rot[i, j]))
            want[r, j] = acc
    assert y.tobytes() == want.tobytes()
    np.testing.assert_allclose(y, x.astype(np.float64) @ rot.astype(np.float64), rtol=0, atol=1e-5)
    # the identity rotates exactly
    assert O.rotate_f32(x, np.eye(24, dtype=np.float32)).tobytes() == x.tobytes()
