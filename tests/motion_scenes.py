"""Scenes and float64 closed forms for the motion-blur tests (test_oracle_motion.py, test_gpu_parity_motion.py).

pan_scene: a matte quad (Kd 0.5) in the plane z = 0 under a distant light that shines along +z, seen at maxdepth 1 by a camera that
slides along x and / or turns about the vertical axis (yaw, degrees: rotation about one fixed axis, which the quaternion slerp turns at
a constant rate).  Every camera ray that hits the quad returns Kd / pi * L * 1, every other one 0, so a sample's radiance follows from
its film position and ray time alone -- computed here in float64 without the oracle's or the library's transform code."""
import numpy as np

from rs_pbrt_b200 import _abi
from rs_pbrt_b200.host import HostScene
from rs_pbrt_b200.scenes import look_at_matrix

EYE_Z = -3.0
L_LIGHT = 2.0
KD = 0.5


def _dir(yaw_deg):
    a = np.radians(yaw_deg)
    return np.array([np.sin(a), 0.0, np.cos(a)])


def pan_scene(xres=16, yres=16, spp=16, x0=-1.5, x1=1.5, shutter=(0.25, 0.75), times=(0.0, 1.0), half=(1.0, 1.0), sampler="sobol", yaw=(0.0, 0.0)):
    h = HostScene()
    m = h.material(_abi.MAT_MATTE, [KD, KD, KD, 0.0])
    hx, hy = half
    P = np.array([[-hx, -hy, 0], [hx, -hy, 0], [hx, hy, 0], [-hx, hy, 0]], np.float32)
    h.trianglemesh(np.array([0, 1, 2, 0, 2, 3], np.uint32), P, material=m)
    h.light_distant([0.0, 0.0, -1.0], [0.0, 0.0, 0.0], [L_LIGHT] * 3)
    e0, e1 = np.array([x0, 0.0, EYE_Z]), np.array([x1, 0.0, EYE_Z])
    h.look_at(e0, e0 + _dir(yaw[0]), [0, 1, 0])
    h.transform_times(*times)
    h.camera_motion(look_at_matrix(e1, e1 + _dir(yaw[1]), [0, 1, 0]))
    h.film(xres, yres)
    h.camera(fov=90.0, shutteropen=shutter[0], shutterclose=shutter[1])
    h.sampler(spp, name=sampler)
    h.integrator(maxdepth=1)
    h.world_end(n_threads=1)
    return h


def eye_x(u, x0, x1, shutter, times):
    """Camera x at camera sample time u: ray.time = lerp(u, shutter) (perspective.rs:226), then the translation lerp of
    AnimatedTransform::interpolate, clamped to the keyframes outside [start_time, end_time]."""
    t = (1.0 - u) * shutter[0] + u * shutter[1]
    dt = np.clip((t - times[0]) / (times[1] - times[0]), 0.0, 1.0)
    return (1.0 - dt) * x0 + dt * x1


def screen(p_film, xres, yres):
    """Film position -> camera-space direction (x, y, 1) of a 90-degree perspective camera (screen window of the aspect ratio)."""
    a = xres / yres
    sw = (-a, a, -1.0, 1.0) if a > 1 else (-1.0, 1.0, -1.0 / a, 1.0 / a)
    sx = sw[0] + p_film[..., 0] / xres * (sw[1] - sw[0])
    sy = sw[3] - p_film[..., 1] / yres * (sw[3] - sw[2])
    return sx, sy


def pan_radiance(p_film, u, xres, yres, x0=-1.5, x1=1.5, shutter=(0.25, 0.75), times=(0.0, 1.0), half=(1.0, 1.0), yaw=(0.0, 0.0)):
    """Expected radiance per sample, and each sample's distance (in the quad's plane) to the nearest quad edge."""
    sx, sy = screen(np.asarray(p_film, np.float64), xres, yres)
    u = np.asarray(u, np.float64)
    a = np.radians(eye_x(u, yaw[0], yaw[1], shutter, times))  # the yaw at the ray's time, lerped like the translation
    # camera x = LookAt's `left` = (cos a, 0, -sin a), y = up, z = (sin a, 0, cos a)
    dx, dz = sx * np.cos(a) + np.sin(a), -sx * np.sin(a) + np.cos(a)
    t = np.where(dz > 0, -EYE_Z / np.where(dz > 0, dz, 1.0), np.inf)
    x = eye_x(u, x0, x1, shutter, times) + t * dx
    y = t * sy
    hit = (dz > 0) & (np.abs(x) <= half[0]) & (np.abs(y) <= half[1])
    edge = np.minimum(np.abs(np.abs(x) - half[0]), np.abs(np.abs(y) - half[1]))
    return np.where(hit, KD / np.pi * L_LIGHT, 0.0), edge


def pan_coverage(px, xres, yres, x0=-1.5, x1=1.5, shutter=(0.25, 0.75), times=(0.0, 1.0), half=1.0, n=4001):
    """Space-time coverage of pixel column px by the quad (rows that see the quad at every x): the share of (film x in the pixel,
    u in [0, 1)) whose ray hits it -- the exact length of the u interval for each film x, averaged over a dense grid of film x."""
    fx = px + (np.arange(n) + 0.5) / n
    sx, _ = screen(np.stack([fx, np.zeros_like(fx)], -1), xres, yres)
    # hit iff |e(u) + 3 sx| <= half, e(u) piecewise linear in u: integrate over u by the same dense rule
    u = (np.arange(n) + 0.5) / n
    e = eye_x(u, x0, x1, shutter, times)
    return float(np.mean(np.abs(e[None, :] + (-EYE_Z) * sx[:, None]) <= half))
