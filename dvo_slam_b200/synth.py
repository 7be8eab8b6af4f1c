"""Seeded analytic RGB-D frame-pair generator (bench/test harness; not on the hot path).

Scene and motion follow SURVEY.md section 8(d): fr1 intrinsics (dvo_benchmark/src/benchmark_slam.cpp:384),
a slanted back plane plus a fronto-parallel box face, albedo = seeded sum of 3-D sinusoids,
depth quantised to 1/5000 m like TUM u16 depth (benchmark_slam.cpp:77), NaN holes, NaN beyond 4 m.
Both cameras ray-cast the same analytic scene, so a true SE(3) exists for every pair:
``p_cur = T_true @ p_ref``.  DenseTracker::match returns ``estimate^-1`` (dense_tracking.cpp:371),
i.e. the expected ``Result.Transformation`` is ``inv(T_true)``.

Runs on any torch device (CPU in the unit tests, CUDA when the bench builds its batch).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace

import numpy as np
import torch

FR1_INTRINSICS = (517.3, 516.5, 318.6, 255.3)  # fx, fy, ox, oy


def se3_exp(xi: np.ndarray) -> np.ndarray:
    """Closed-form SE(3) exponential, twist order [v; omega] (Sophus convention)."""
    xi = np.asarray(xi, dtype=np.float64)
    v, w = xi[:3], xi[3:]
    th = float(np.linalg.norm(w))
    O = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], dtype=np.float64)
    if th < 1e-10:
        R = np.eye(3) + O
        V = np.eye(3) + 0.5 * O
    else:
        R = np.eye(3) + math.sin(th) / th * O + (1 - math.cos(th)) / th**2 * (O @ O)
        V = np.eye(3) + (1 - math.cos(th)) / th**2 * O + (th - math.sin(th)) / th**3 * (O @ O)
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = V @ v
    return T


def se3_log(T: np.ndarray) -> np.ndarray:
    R, t = T[:3, :3], T[:3, 3]
    c = max(-1.0, min(1.0, (np.trace(R) - 1) / 2))
    th = math.acos(c)
    if th < 1e-10:
        w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
        Vi = np.eye(3)
    else:
        w = th / (2 * math.sin(th)) * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
        O = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        Vi = np.eye(3) - 0.5 * O + (1 - th * math.cos(th / 2) / (2 * math.sin(th / 2))) / th**2 * (O @ O)
    return np.concatenate([Vi @ t, w])


@dataclass
class SceneConfig:
    width: int = 640
    height: int = 480
    intrinsics: tuple = FR1_INTRINSICS
    n_sinusoids: int = 32
    max_translation: float = 0.03   # metres per axis
    max_rotation: float = 0.02      # radians per axis
    hole_fraction: float = 0.03     # fraction of 8x8 blocks set to NaN depth
    max_depth: float = 4.0
    depth_quantum: float = 1.0 / 5000.0
    intensity_noise_sigma: float = 0.0
    quantize_intensity: bool = True
    distortion: tuple | None = None  # (k1, k2, p1, p2, k3) plumb-bob lens; None: a pinhole camera
    depth_camera: "DepthCamera | None" = None   # depth from a camera of its own; None: depth along the colour rays

    def scaled(self, factor: int) -> "SceneConfig":
        """Same camera at ``factor`` x the resolution (config 5: 1280x960 = 2 x fr1)."""
        fx, fy, ox, oy = self.intrinsics
        return SceneConfig(self.width * factor, self.height * factor,
                           (fx * factor, fy * factor, ox * factor, oy * factor), self.n_sinusoids,
                           self.max_translation, self.max_rotation, self.hole_fraction, self.max_depth,
                           self.depth_quantum, self.intensity_noise_sigma, self.quantize_intensity, self.distortion,
                           self.depth_camera)


@dataclass
class DepthCamera:
    """A depth camera apart from the colour camera (a time-of-flight or stereo depth sensor): its own size, intrinsics and
    optional plumb-bob distortion, at T_color_depth (4x4, p_color = T_color_depth @ p_depth, metres)."""
    width: int
    height: int
    intrinsics: tuple
    T_color_depth: np.ndarray
    distortion: tuple | None = None


def baseline(tx: float, ty: float = 0.0, tz: float = 0.0) -> np.ndarray:
    """T_color_depth of a depth camera mounted parallel to the colour camera at (tx, ty, tz) metres in its frame"""
    T = np.eye(4)
    T[:3, 3] = (tx, ty, tz)
    return T


FR1_DISTORTION = (0.2624, -0.9531, -0.0054, 0.0026, 1.1633)   # TUM fr1 plumb-bob k1, k2, p1, p2, k3


def undistort_points(xd, yd, dist, tol: float = 1e-12, max_iter: int = 100):
    """Normalised pinhole coordinates (x, y) whose plumb-bob distortion (OpenCV's model, dist = (k1, k2, p1, p2, k3)) is
    (xd, yd): Newton's method in float64 from (xd, yd) until the residual is below tol."""
    k1, k2, p1, p2, k3 = (float(v) for v in dist)
    x, y = xd.clone(), yd.clone()
    for _ in range(max_iter):
        r2 = x * x + y * y
        R = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
        dR = k1 + (2 * k2 + 3 * k3 * r2) * r2           # dR / dr2
        fx = x * R + 2 * p1 * x * y + p2 * (r2 + 2 * x * x) - xd
        fy = y * R + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y - yd
        if max(float(fx.abs().max()), float(fy.abs().max())) < tol:
            return x, y
        a = R + 2 * x * x * dR + 2 * p1 * y + 6 * p2 * x  # Jacobian [[a, b], [c, d]]
        b = 2 * x * y * dR + 2 * p1 * x + 2 * p2 * y
        d = R + 2 * y * y * dR + 6 * p1 * y + 2 * p2 * x
        det = a * d - b * b
        x, y = x - (d * fx - b * fy) / det, y - (a * fy - b * fx) / det
    raise RuntimeError(f"undistort_points: no convergence to {tol} in {max_iter} iterations")


def _render(cfg: SceneConfig, T_cam: np.ndarray, tex, box, rng: np.random.Generator, device):
    """Ray-cast the scene from a camera whose pose satisfies p_cam = T_cam @ p_ref."""
    f64 = torch.float64
    fx, fy, ox, oy = cfg.intrinsics
    w, h = cfg.width, cfg.height
    T = torch.tensor(T_cam, dtype=f64, device=device)
    R, t = T[:3, :3], T[:3, 3]
    xs = (torch.arange(w, dtype=f64, device=device) - ox) / fx
    ys = (torch.arange(h, dtype=f64, device=device) - oy) / fy
    xs, ys = xs[None, :].expand(h, w), ys[:, None].expand(h, w)
    if cfg.distortion is not None:   # pixel (u, v) of the lens sees the ray of the pinhole point it distorts from
        xs, ys = undistort_points(xs.contiguous(), ys.contiguous(), cfg.distortion)
    dc = torch.stack([xs, ys, torch.ones(h, w, dtype=f64, device=device)], -1)   # d_cam.z = 1: depth stays the z-distance
    d = dc @ R            # rows: R^T d_cam  (direction in the reference frame)
    o = -(R.T @ t)        # camera centre in the reference frame
    # back plane: z - 0.3x - 0.2y = 2.5
    nb = torch.tensor([-0.3, -0.2, 1.0], dtype=f64, device=device)
    s_back = (2.5 - (nb * o).sum()) / (d * nb).sum(-1)
    # box face: z = zb, |x-cx|<=ax, |y-cy|<=ay
    zb, cx, cy, ax, ay = box
    s_box = (zb - o[2]) / d[..., 2]
    hit = o + s_box[..., None] * d
    in_box = (s_box > 0) & ((hit[..., 0] - cx).abs() <= ax) & ((hit[..., 1] - cy).abs() <= ay)
    s = torch.where(in_box & (s_box < s_back), s_box, s_back)
    X = o + s[..., None] * d                       # surface point, reference frame
    depth = s * 1.0                                 # z in the camera frame: d_cam.z == 1
    # albedo: sum of 3-D sinusoids
    freq, phase, amp = tex
    arg = 2 * math.pi * (X.reshape(-1, 3) @ freq.T) + phase
    val = (torch.sin(arg) * amp).sum(-1).reshape(h, w)
    inten = 127.5 + 107.5 * torch.clamp(val, -1.0, 1.0)
    if cfg.intensity_noise_sigma > 0:
        noise = torch.tensor(rng.standard_normal((h, w)), dtype=f64, device=device)
        inten = inten + cfg.intensity_noise_sigma * noise
    if cfg.quantize_intensity:
        inten = torch.round(inten)
    inten = torch.clamp(inten, 0.0, 255.0)
    depth = torch.round(depth / cfg.depth_quantum) * cfg.depth_quantum
    depth = torch.where((depth > cfg.max_depth) | (s <= 0), torch.full_like(depth, float("nan")), depth)
    # NaN holes: seeded 8x8 blocks
    hb, wb = (h + 7) // 8, (w + 7) // 8
    holes = torch.tensor(rng.random((hb, wb)) < cfg.hole_fraction, device=device)
    holes = holes.repeat_interleave(8, 0).repeat_interleave(8, 1)[:h, :w]
    depth = torch.where(holes, torch.full_like(depth, float("nan")), depth)
    return inten.to(torch.float32), depth.to(torch.float32)


def make_pair(seed: int, cfg: SceneConfig | None = None, device="cpu"):
    """Returns dict with float32 [h,w] tensors I_ref, Z_ref, I_cur, Z_cur on ``device`` and
    float64 numpy ``T_true`` (p_cur = T_true p_ref) and ``xi``.  With ``cfg.depth_camera``, Z_ref / Z_cur are that camera's
    depth frames in its own geometry, and Z_ref_color / Z_cur_color the colour camera's own depth."""
    cfg = cfg or SceneConfig()
    rng = np.random.default_rng(seed)
    xi = np.concatenate([rng.uniform(-cfg.max_translation, cfg.max_translation, 3),
                         rng.uniform(-cfg.max_rotation, cfg.max_rotation, 3)])
    T_true = se3_exp(xi)
    # texture: wavelengths 4..60 cm, amplitude ~ wavelength (coarse structure dominates)
    lam = np.exp(rng.uniform(math.log(0.04), math.log(0.60), cfg.n_sinusoids))
    dirs = rng.standard_normal((cfg.n_sinusoids, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    freq = dirs / lam[:, None]
    phase = rng.uniform(0, 2 * math.pi, cfg.n_sinusoids)
    amp = lam / lam.sum() * 2.2
    f64 = torch.float64
    tex = (torch.tensor(freq, dtype=f64, device=device), torch.tensor(phase, dtype=f64, device=device),
           torch.tensor(amp, dtype=f64, device=device))
    box = (1.2 + rng.uniform(-0.1, 0.1), rng.uniform(-0.2, 0.2), rng.uniform(-0.15, 0.15), 0.28, 0.22)
    I_ref, Z_ref = _render(cfg, np.eye(4), tex, box, rng, device)
    I_cur, Z_cur = _render(cfg, T_true, tex, box, rng, device)
    out = {"I_ref": I_ref, "Z_ref": Z_ref, "I_cur": I_cur, "Z_cur": Z_cur, "T_true": T_true, "xi": xi,
           "intrinsics": cfg.intrinsics, "width": cfg.width, "height": cfg.height}
    if cfg.depth_camera is not None:
        # Z_ref / Z_cur come from the depth camera, in its own geometry, after the colour frames have drawn from rng;
        # the colour camera's own depth stays as Z_ref_color / Z_cur_color
        dc = cfg.depth_camera
        dcfg = replace(cfg, width=dc.width, height=dc.height, intrinsics=tuple(dc.intrinsics), distortion=dc.distortion,
                       depth_camera=None)
        T_dc = np.linalg.inv(np.asarray(dc.T_color_depth, dtype=np.float64))   # p_depth = T_dc p_color
        out["Z_ref_color"], out["Z_cur_color"] = Z_ref, Z_cur
        out["Z_ref"] = _render(dcfg, T_dc, tex, box, rng, device)[1]
        out["Z_cur"] = _render(dcfg, T_dc @ T_true, tex, box, rng, device)[1]
    return out


def make_sequence(seed: int, n_frames: int, cfg: SceneConfig | None = None, device="cpu"):
    """A camera moving through one scene: returns (frames, poses) with frames[k] = (I, Z) float32 tensors and
    poses[k] the float64 4x4 world-from-camera pose of frame k (frame 0 = identity).  Consecutive frames differ
    by a twist drawn like make_pair's, so relative_k = poses[k-1]^-1 poses[k] is what DenseTracker::match returns
    for (reference = frame k-1, current = frame k)."""
    cfg = cfg or SceneConfig()
    rng = np.random.default_rng(seed)
    lam = np.exp(rng.uniform(math.log(0.04), math.log(0.60), cfg.n_sinusoids))
    dirs = rng.standard_normal((cfg.n_sinusoids, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    f64 = torch.float64
    tex = (torch.tensor(dirs / lam[:, None], dtype=f64, device=device),
           torch.tensor(rng.uniform(0, 2 * math.pi, cfg.n_sinusoids), dtype=f64, device=device),
           torch.tensor(lam / lam.sum() * 2.2, dtype=f64, device=device))
    box = (1.2 + rng.uniform(-0.1, 0.1), rng.uniform(-0.2, 0.2), rng.uniform(-0.15, 0.15), 0.28, 0.22)
    T_cam = np.eye(4)            # p_cam = T_cam p_world
    frames, poses = [], []
    for k in range(n_frames):
        if k > 0:
            xi = np.concatenate([rng.uniform(-cfg.max_translation, cfg.max_translation, 3),
                                 rng.uniform(-cfg.max_rotation, cfg.max_rotation, 3)])
            T_cam = se3_exp(xi) @ T_cam
        frames.append(_render(cfg, T_cam, tex, box, rng, device))
        poses.append(np.linalg.inv(T_cam))
    return frames, poses


def _patch_texture(rng, pw: int, ph: int, amplitude: float) -> np.ndarray:
    """A (ph, pw) float32 texture of twelve random plane waves around mid-grey, rounded to 8-bit levels."""
    yy, xx = np.mgrid[0:ph, 0:pw]
    tex = np.zeros((ph, pw))
    for _ in range(12):
        kx, ky = rng.uniform(-0.25, 0.25, 2)
        tex += rng.uniform(0.3, 1.0) * np.sin(kx * xx + ky * yy + rng.uniform(0, 2 * math.pi))
    return np.round(np.clip(127.5 + amplitude * tex, 0, 255)).astype(np.float32)


def make_moving_object_pair(seed: int, cfg: SceneConfig | None = None, patch=(150, 120), corner=(250, 200), shift=(24, 10),
                            z_obj: float = 0.9, margin: int = 8):
    """make_pair plus an object that moves on its own: a textured fronto-parallel patch (patch = (w, h) pixels at depth
    ~z_obj, the size of a person at ~1 m) pasted at corner = (x, y) in the reference frame and at corner + shift in the
    current frame, whatever the camera did.  Returns make_pair's dict (float32 numpy images, T_true of the camera) plus
    "mask": the uint8 reference mask that excludes the patch and a margin of `margin` pixels around it (0 = excluded),
    as a dilated segmentation mask would."""
    p = make_pair(seed, cfg)
    out = dict(p)
    for k in ("I_ref", "Z_ref", "I_cur", "Z_cur"):
        out[k] = p[k].cpu().numpy().copy()
    rng = np.random.default_rng(1000 + seed)
    pw, ph = patch
    yy, xx = np.mgrid[0:ph, 0:pw]
    tex = _patch_texture(rng, pw, ph, 40.0)
    zt = (np.float32(z_obj) + np.float32(0.0002) * np.round(xx / 8.0)).astype(np.float32)
    x0, y0 = corner
    x1, y1 = x0 + shift[0], y0 + shift[1]
    out["I_ref"][y0:y0 + ph, x0:x0 + pw] = tex
    out["Z_ref"][y0:y0 + ph, x0:x0 + pw] = zt
    out["I_cur"][y1:y1 + ph, x1:x1 + pw] = tex
    out["Z_cur"][y1:y1 + ph, x1:x1 + pw] = zt
    mask = np.ones(out["I_ref"].shape, np.uint8)
    mask[max(y0 - margin, 0):y0 + ph + margin, max(x0 - margin, 0):x0 + pw + margin] = 0
    out["mask"] = mask
    return out


def make_overlay_pair(seed: int, size=(160, 120), corner=(420, 300), margin: int = 8, cfg: SceneConfig | None = None):
    """make_pair plus a textured overlay fixed in the image: size = (w, h) pixels at corner = (x, y), written into the
    intensity of BOTH frames at the same position, with the scene's depth left as it is -- a logo or timestamp burnt into
    the colour image, a lens smudge or a glare patch.  Its pixels have the right depth and the wrong intensity, so the
    occlusion test cannot reject taps on them.  Returns make_pair's dict (float32 numpy images, T_true of the camera) plus
    "mask": the uint8 mask of either frame that excludes the overlay and a margin of `margin` pixels around it (0 =
    excluded)."""
    p = make_pair(seed, cfg)
    out = dict(p)
    for k in ("I_ref", "Z_ref", "I_cur", "Z_cur"):
        out[k] = p[k].cpu().numpy().copy()
    pw, ph = size
    tex = _patch_texture(np.random.default_rng(2000 + seed), pw, ph, 60.0)
    x0, y0 = corner
    out["I_ref"][y0:y0 + ph, x0:x0 + pw] = tex[:out["I_ref"].shape[0] - y0, :out["I_ref"].shape[1] - x0]
    out["I_cur"][y0:y0 + ph, x0:x0 + pw] = tex[:out["I_cur"].shape[0] - y0, :out["I_cur"].shape[1] - x0]
    mask = np.ones(out["I_ref"].shape, np.uint8)
    mask[max(y0 - margin, 0):y0 + ph + margin, max(x0 - margin, 0):x0 + pw + margin] = 0
    out["mask"] = mask
    return out


def exposure(I, gain: float, bias: float):
    """An auto-exposure / white-balance change of a frame: clip(round(gain I + bias), 0, 255), in float32 arithmetic (gain and
    bias rounded to float32, ties to even)."""
    I = np.asarray(I, dtype=np.float32)
    return np.clip(np.round(np.float32(gain) * I + np.float32(bias)), 0, 255).astype(np.float32)
