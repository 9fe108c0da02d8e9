"""The three quaternion helpers of trimesh.transformations that make_dataset.py:sample_blensor and _pcd_files_to_pts
use (make_dataset.py:203,315), restated from the published formulas.  Quaternions are [w, x, y, z]."""
import numpy as np

_EPS = np.finfo(float).eps * 4.0


def random_quaternion(rand=None):
    """Uniformly distributed unit quaternion from three uniforms in [0, 1) (Shoemake, "Uniform random rotations",
    Graphics Gems III, 1992)."""
    if rand is None:
        rand = np.random.rand(3)
    else:
        assert len(rand) == 3
    r1 = np.sqrt(1.0 - rand[0])
    r2 = np.sqrt(rand[0])
    t1 = 2.0 * np.pi * rand[1]
    t2 = 2.0 * np.pi * rand[2]
    return np.array([np.cos(t2) * r2, np.sin(t1) * r1, np.cos(t1) * r1, np.sin(t2) * r2])


def quaternion_matrix(quaternion):
    """4x4 homogeneous rotation matrix of a quaternion (normalised first; identity for a near-zero quaternion)."""
    q = np.array(quaternion, dtype=np.float64, copy=True)
    n = np.dot(q, q)
    if n < _EPS:
        return np.identity(4)
    q *= np.sqrt(2.0 / n)
    q = np.outer(q, q)
    return np.array([
        [1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0], 0.0],
        [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0], 0.0],
        [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2], 0.0],
        [0.0, 0.0, 0.0, 1.0]])


def quaternion_conjugate(quaternion):
    """[w, -x, -y, -z]: the inverse rotation of a unit quaternion."""
    q = np.array(quaternion, dtype=np.float64, copy=True)
    np.negative(q[1:], q[1:])
    return q
