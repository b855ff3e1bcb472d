"""Camera paths of the reference's validation videos, on the host in fp64:

* get_turntable_cameras (diffusionGS/models/gsrenderer/gs_core.py:49-85): the object model's turntable;
* get_interpolated_poses_many (diffusionGS/models/gsrenderer/cam_utils.py:105-278): the scene model's keyframe
  fly-through, rotations by quaternion slerp and positions and intrinsics blended linearly.

Both are a few hundred 4x4 matrices, so they are built with numpy scalar arithmetic, operation for operation as the
reference builds them: the cameras, and so the frames, are the reference's to the last bit.
"""
import math

import numpy as np
import torch

_EPS = np.finfo(float).eps * 4.0  # the slerp's tolerance (cam_utils.py:28)


def get_turntable_cameras(hfov=50, num_views=8, w=384, h=384, radius=2.7, elevation=0, up_vector=(0, 0, 1)):
    """-> (w, h, num_views, fxfycxcy fp64 [num_views, 4], c2ws fp64 [num_views, 4, 4]): OpenCV-convention cameras
    (x right, y down, z forward) at `radius` around the origin, `elevation` degrees above the xy plane, at azimuths
    linspace(0, 360, num_views, endpoint=False), each looking at the origin."""
    fx = w / (2 * np.tan(np.deg2rad(hfov) / 2.0))
    fxfycxcy = np.array([fx, fx, w / 2.0, h / 2.0]).reshape(1, 4).repeat(num_views, axis=0)
    azimuths = np.linspace(0, 360, num_views, endpoint=False)
    c2ws = np.zeros((num_views, 4, 4))
    for i, azim in enumerate(azimuths):
        el, az = np.deg2rad(elevation), np.deg2rad(azim)
        ring = radius * np.cos(el)
        pos = np.array([ring * np.cos(az), ring * np.sin(az), radius * np.sin(el)])
        fwd = -pos / np.linalg.norm(pos)
        right = np.cross(fwd, up_vector)
        right = right / np.linalg.norm(right)
        up = np.cross(right, fwd)
        up = up / np.linalg.norm(up)
        c2ws[i] = np.eye(4)
        c2ws[i, :3, 0], c2ws[i, :3, 1], c2ws[i, :3, 2], c2ws[i, :3, 3] = right, -up, fwd, pos
    return w, h, num_views, fxfycxcy, c2ws


def sphere_cameras(num_views=100, image_size=512):
    """-> (fxfycxcy fp64 [n, 4], c2ws fp64 [n, 4, 4]): OpenCV-convention cameras (as get_turntable_cameras) on the
    sphere of radius 4, each looking at the origin.  View k looks from the Fibonacci-sphere direction with
    z = 1 - (2k + 1) / n at azimuth k * pi * (3 - sqrt(5)), with +z up (+y where the direction is within 0.99 of +-z).
    The images are square, image_size pixels wide, with the half-angle asin(sqrt(3) / 4): the sphere around the cube
    [-1, 1]^3 just fits in every view."""
    n, s = int(num_views), float(image_size)
    fx = s / (2 * math.tan(math.asin(math.sqrt(3.0) / 4)))
    fxfycxcy = np.array([fx, fx, s / 2.0, s / 2.0]).reshape(1, 4).repeat(n, axis=0)
    c2ws = np.zeros((n, 4, 4))
    for k in range(n):
        z = 1 - (2 * k + 1) / n
        ring, az = math.sqrt(max(0.0, 1 - z * z)), k * math.pi * (3 - math.sqrt(5))
        d = np.array([ring * math.cos(az), ring * math.sin(az), z])
        fwd = -d
        right = np.cross(fwd, (0.0, 1.0, 0.0) if abs(z) > 0.99 else (0.0, 0.0, 1.0))
        right = right / np.linalg.norm(right)
        up = np.cross(right, fwd)
        up = up / np.linalg.norm(up)
        c2ws[k] = np.eye(4)
        c2ws[k, :3, 0], c2ws[k, :3, 1], c2ws[k, :3, 2], c2ws[k, :3, 3] = right, -up, fwd, 4 * d
    return fxfycxcy, c2ws


def _unit(q):
    q = np.array(q, dtype=np.float64)
    return q / math.sqrt(np.dot(q, q))


def _quaternion(R):
    """Unit quaternion (w, x, y, z), w >= 0, of the rotation R [3, 3]: the eigenvector of the largest eigenvalue of
    Bar-Itzhack's symmetric 4x4 matrix, which tolerates a slightly non-orthogonal R."""
    m = np.asarray(R, dtype=np.float64)
    K = np.array([
        [m[0, 0] - m[1, 1] - m[2, 2], 0.0, 0.0, 0.0],
        [m[0, 1] + m[1, 0], m[1, 1] - m[0, 0] - m[2, 2], 0.0, 0.0],
        [m[0, 2] + m[2, 0], m[1, 2] + m[2, 1], m[2, 2] - m[0, 0] - m[1, 1], 0.0],
        [m[2, 1] - m[1, 2], m[0, 2] - m[2, 0], m[1, 0] - m[0, 1], m[0, 0] + m[1, 1] + m[2, 2]],
    ])
    K /= 3.0
    evals, evecs = np.linalg.eigh(K)  # reads the lower triangle
    q = evecs[np.array([3, 0, 1, 2]), np.argmax(evals)]
    return -q if q[0] < 0.0 else q


def _slerp(qa, qb, t):
    """Spherical interpolation from qa (t = 0) to qb (t = 1) along the shorter arc."""
    q0, q1 = _unit(qa), _unit(qb)
    if t == 0.0:
        return q0
    if t == 1.0:
        return q1
    d = np.dot(q0, q1)
    if abs(abs(d) - 1.0) < _EPS:  # the same rotation
        return q0
    if d < 0.0:  # q and -q are one rotation: take the shorter way round
        d, q1 = -d, -q1
    angle = math.acos(d)
    if abs(angle) < _EPS:
        return q0
    inv_sin = 1.0 / math.sin(angle)
    return q0 * (math.sin((1.0 - t) * angle) * inv_sin) + q1 * (math.sin(t * angle) * inv_sin)


def _rotation(q):
    """Rotation matrix [3, 3] of the quaternion q (w, x, y, z), normalised on the way; identity for a null q."""
    q = np.array(q, dtype=np.float64)
    n = np.dot(q, q)
    if n < _EPS:
        return np.identity(3)
    q = np.outer(q * math.sqrt(2.0 / n), q * math.sqrt(2.0 / n))
    return np.array([
        [1.0 - q[2, 2] - q[3, 3], q[1, 2] - q[3, 0], q[1, 3] + q[2, 0]],
        [q[1, 2] + q[3, 0], 1.0 - q[1, 1] - q[3, 3], q[2, 3] - q[1, 0]],
        [q[1, 3] - q[2, 0], q[2, 3] + q[1, 0], 1.0 - q[1, 1] - q[2, 2]],
    ])


def get_interpolated_poses_many(poses, Ks, steps_per_transition=10, order_poses=False):
    """poses [n, 3, 4] camera-to-world, Ks [n, 3, 3] tensors -> (poses [(n-1) * steps, 3, 4] on the CPU,
    Ks [(n-1) * steps, 3, 3] on the device of `Ks`), fp32.  Every transition a -> b contributes `steps_per_transition`
    cameras at t = linspace(0, 1, steps), both ends included, so the camera where two transitions meet appears twice,
    as in the reference.  Rotations follow
    the shortest-arc slerp of their quaternions, positions the straight line, both in fp64; the intrinsics are blended
    as Ks[a] * (1 - t) + Ks[b] * t in the dtype of `Ks`.  order_poses=True (the reference's nearest-neighbour
    reordering) has no caller and is not supported."""
    if order_poses:
        raise NotImplementedError("order_poses=True is not supported: pass the keyframes in the order to visit them")
    poses64 = np.asarray(poses.detach().cpu().numpy() if torch.is_tensor(poses) else poses, dtype=np.float64)
    ts = np.linspace(0, 1, steps_per_transition)
    traj, k_interp = [], []
    for a in range(poses64.shape[0] - 1):
        pa, pb = poses64[a], poses64[a + 1]
        qa, qb = _quaternion(pa[:3, :3]), _quaternion(pb[:3, :3])
        for t in ts:
            pose = np.zeros((3, 4))
            pose[:, :3] = _rotation(_slerp(qa, qb, t))
            pose[:, 3] = (1 - t) * pa[:3, 3] + t * pb[:3, 3]
            traj.append(pose)
            k_interp.append(Ks[a] * (1.0 - t) + Ks[a + 1] * t)
    return torch.tensor(np.stack(traj), dtype=torch.float32), torch.stack(k_interp).to(torch.float32)
