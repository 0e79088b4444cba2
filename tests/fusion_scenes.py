"""Seeded analytic scenes for the fusion tests: depth maps ray-cast in fp64 from planes and spheres, with poses and colours."""
import numpy as np


def look_at(eye, target, up=(0.0, -1.0, 0.0)):
    """Camera-to-world [4,4] of a camera at eye looking at target (camera x right, y down, z forward)."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(-np.asarray(up, np.float64), z)
    if np.linalg.norm(x) < 1e-6:
        x = np.cross((1.0, 0.0, 0.0), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4)
    T[:3, :3] = np.stack([x, y, z], 1)
    T[:3, 3] = eye
    return T


def render(K, T, H, W, planes=(), spheres=()):
    """Depth [H,W] (camera z) of the nearest surface along each pixel centre's ray, 0 where no surface is hit.
    planes: (normal n, offset c) with n . p = c; spheres: (centre, radius)."""
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    d_cam = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)
    d = d_cam @ T[:3, :3].T
    o = T[:3, 3]
    best = np.full((H, W), np.inf)
    for n, c in planes:
        n = np.asarray(n, np.float64)
        den = d @ n
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (c - o @ n) / den
        best = np.where((t > 0) & (t < best), t, best)
    for ctr, r in spheres:
        oc = o - np.asarray(ctr, np.float64)
        a = np.sum(d * d, -1)
        b = 2 * d @ oc
        cc = oc @ oc - r * r
        disc = b * b - 4 * a * cc
        t = (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a)
        best = np.where((disc >= 0) & (t > 0) & (t < best), t, best)
    return np.where(np.isfinite(best), best, 0.0)


def street(seed, n_frames, H=48, W=64):
    """Frames of a small street: a ground plane, a back wall, a side wall and two spheres, seen from cameras moving forward
    with small turns.  Returns (depth [F,H,W] float32 with noise and 0 / NaN / far pixels, colour [F,H,W,3] uint8,
    K [F,3,3] (two focal lengths), cam_to_world [F,4,4])."""
    rng = np.random.default_rng(seed)
    planes = [((0.0, 1.0, 0.0), 1.1), ((0.0, 0.0, 1.0), 4.7), ((1.0, 0.0, 0.0), 1.7)]
    spheres = [((0.25, 0.3, 2.6), 0.55), ((-0.9, 0.6, 3.4), 0.4)]
    depth, color, Ks, Ts = [], [], [], []
    for f in range(n_frames):
        fx = 46.0 if f % 3 else 52.5
        K = np.array([[fx, 0, (W - 1) / 2 + 0.3], [0, fx * 1.02, (H - 1) / 2 - 0.2], [0, 0, 1]])
        eye = np.array([-0.3 + 0.04 * f, -0.1 + 0.02 * np.sin(f), 0.2 + 0.08 * f]) + rng.normal(0, 0.01, 3)
        target = np.array([0.2 * np.cos(0.4 * f), 0.2, 3.5]) + rng.normal(0, 0.05, 3)
        T = look_at(eye, target)
        d = render(K, T, H, W, planes, spheres)
        d = d * (1 + rng.normal(0, 2e-3, d.shape))
        flat = d.reshape(-1)
        idx = rng.choice(flat.size, 12, replace=False)
        flat[idx[:4]] = 0.0
        flat[idx[4:8]] = np.nan
        flat[idx[8:]] = 60.0
        depth.append(d.astype(np.float32))
        color.append(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        Ks.append(K)
        Ts.append(T)
    return np.stack(depth), np.stack(color), np.stack(Ks), np.stack(Ts)


def sphere_views(centre, radius, n=12, dist=2.5, H=192, W=192, f=180.0):
    """Depth maps of one sphere from n directions spread over the sphere (a Fibonacci lattice), background 0."""
    K = np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]])
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = np.pi * (1 + 5 ** 0.5) * i
    dirs = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
    Ts = np.stack([look_at(np.asarray(centre) + dist * dv, centre, up=(0.3, -1.0, 0.2)) for dv in dirs])
    depth = np.stack([render(K, T, H, W, spheres=[(centre, radius)]) for T in Ts]).astype(np.float32)
    return depth, K, Ts
