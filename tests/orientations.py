"""The camera orientations the orientation tests run at (tests/test_host_orientations.py, tests/test_gpu_orientations.py,
the rotated fixtures of tests/golden/make_ref_golden.py).

make_scene's own ground truths stay within 30 degrees of the world axes; real cameras do not.  The set below covers the
identity, quarter turns, the approach to a half turn, exact half turns (where Rodrigues' matrix -> vector conversion takes
its separate branch) and a few rotations drawn uniformly over SO(3).  Each entry is a world->camera rotation matrix
(float64).  Half turns are built as 2 k k^T - I, which is exact for the axis-aligned k: diag(1, -1, -1) is a camera with
y down looking along world -z in a world with y up.
"""
import numpy as np

from esac_b200.synth import rodrigues

N_AXIS = np.array([1.0, 2.0, 3.0]) / np.sqrt(14.0)
# the only axis of the set for which the near-pi branch flips the sign of z: x = 0, and y, z of opposite signs
YZ_AXIS = np.array([0.0, 2.0, -3.0]) / np.sqrt(13.0)


def half_turn(axis) -> np.ndarray:
    k = np.asarray(axis, np.float64).reshape(3, 1)
    return 2.0 * (k @ k.T) - np.eye(3)


def uniform_rotations(n: int, seed: int = 2024) -> list:
    """n rotations uniform over SO(3): unit quaternions from normalised 4-d Gaussians."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        q = rng.normal(size=4)
        w, x, y, z = q / np.linalg.norm(q)
        out.append(np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                             [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                             [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]))
    return out


def _set() -> dict:
    e = np.eye(3)
    s = {"identity": np.eye(3)}
    for name, ax in (("x", e[0]), ("y", e[1]), ("z", e[2]), ("n", N_AXIS)):
        s[f"90_{name}"] = rodrigues(ax * (np.pi / 2))
    for name, ang in (("150", np.radians(150.0)), ("179", np.radians(179.0)), ("179.99", np.radians(179.99)),
                      ("pi-1e-6", np.pi - 1e-6)):
        s[f"{name}_n"] = rodrigues(N_AXIS * ang)
    for name, ax in (("x", e[0]), ("y", e[1]), ("z", e[2]), ("n", N_AXIS), ("0,2,-3", YZ_AXIS)):
        s[f"pi_{name}"] = half_turn(ax)
    for i, R in enumerate(uniform_rotations(5)):
        s[f"uniform{i}"] = R
    return s


ORIENTATIONS = _set()
NAMES = list(ORIENTATIONS)


def rotate(R: np.ndarray, axis, angle: float) -> np.ndarray:
    """R followed by a turn of `angle` about `axis` (a rotation `angle` away from R)."""
    return rodrigues(np.asarray(axis, np.float64) / np.linalg.norm(axis) * angle) @ R


def cam_to_world(R: np.ndarray, centre=(0.3, -0.2, 1.5)) -> np.ndarray:
    """float32 camera->world 4x4 of a camera with world->camera rotation R at `centre` (what gtPose holds)."""
    T = np.eye(4)
    T[:3, :3] = R.T
    T[:3, 3] = centre
    return T.astype(np.float32)
