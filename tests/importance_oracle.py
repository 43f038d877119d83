"""NumPy restatement of the Immersive dataset's importance subsample (hr_build_importance_table, csrc/hr_train_batch.cu), and
the seeded test videos of tests/golden/reference/train_importance.npz.  TEST INFRASTRUCTURE.

ImmersiveDataset.importance_subsample (datasets/immersive.py:295-321): of a frame of N pixels, keep those with diff > thr and
dz < -0.05 in row-major order, diff = mean(|rgb - last_rgb|, -1) of the ToTensor colours (u8 / 255 in fp32; torch evaluates the
mean as ((d0 + d1) + d2) / 3), thr = sort(diff)[-num_take] = the value of ascending rank (N - num_take) % N, dz the ray
direction's z.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence, Tuple

import numpy as np

_M64 = (1 << 64) - 1


def _mix64(z: np.ndarray) -> np.ndarray:
    """The splitmix64 finaliser over uint64 arrays (wrapping arithmetic)."""
    z = z.astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def video_frames(seed: int, n_frames: int, height: int, width: int, static: Sequence[int] = ()) -> np.ndarray:
    """uint8 [n_frames, H, W, 3]: a hashed base image, then per frame a change of -3..3 levels per channel (many equal diffs,
    so ties straddle the threshold) and one pixel in 64 changed by up to 99 levels.  A frame listed in ``static`` repeats its
    predecessor.  Integer hashing only: the same bytes on every machine."""
    n = height * width * 3
    idx = np.arange(n, dtype=np.uint64)
    key = lambda f: np.uint64((int(seed) * 0x9E3779B97F4A7C15 + (f + 1) * 0xD1B54A32D192ED03) & _M64)  # noqa: E731
    cur = (_mix64(idx ^ key(-1)) % np.uint64(256)).astype(np.int64)
    out = []
    for f in range(n_frames):
        if f > 0 and f not in static:
            h = _mix64(idx ^ key(f))
            step = (h % np.uint64(7)).astype(np.int64) - 3
            big = ((h >> np.uint64(8)) % np.uint64(64)) == 0
            jump = ((h >> np.uint64(16)) % np.uint64(199)).astype(np.int64) - 99
            cur = np.clip(cur + np.where(big, jump, step), 0, 255)
        out.append(cur.astype(np.uint8).reshape(height, width, 3))
    return np.stack(out)


def diff_key(cur: np.ndarray, prev: np.ndarray) -> np.ndarray:
    """mean(|cur - prev|, -1) of u8 / 255 colours in fp32, in torch's order ((d0 + d1) + d2) / 3.  cur, prev: uint8 [..., 3]."""
    a = cur.astype(np.float32) / np.float32(255.0)
    b = prev.astype(np.float32) / np.float32(255.0)
    d = np.abs(a - b)
    return ((d[..., 0] + d[..., 1]) + d[..., 2]) / np.float32(3.0)


def keep_mask(cur: np.ndarray, prev: np.ndarray, dz: np.ndarray, num_take: int) -> np.ndarray:
    """importance_subsample's mask of one frame: cur, prev uint8 [H, W, 3] (or [N, 3]), dz fp32 [N]; bool [N]."""
    diff = diff_key(cur, prev).reshape(-1)
    n = diff.shape[0]
    thr = np.sort(diff)[(n - int(num_take)) % n]  # sorted[-num_take], num_take = 0 included
    return (diff > thr) & (np.asarray(dz, dtype=np.float32).reshape(-1) < np.float32(-0.05))


def table_ids(images: np.ndarray, dz: np.ndarray, plan: Sequence[Optional[Tuple[int, int]]]) -> np.ndarray:
    """The table's pixel ids (view*H*W + y*W + x) in table order: images uint8 [n, H, W, 3], dz fp32 [n, H*W] (each view's
    ray z), plan as importance_subsample_plan returns it."""
    n, H, W = images.shape[:3]
    ids = []
    for v, e in enumerate(plan):
        if e is None:
            keep = np.ones(H * W, dtype=bool)
        else:
            take, prev = e
            keep = keep_mask(images[v], images[prev], dz[v], take)
        ids.append(v * H * W + np.flatnonzero(keep))
    return np.concatenate(ids).astype(np.int64)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "train_importance.npz")


def golden_cases():
    """The cases of tests/golden/reference/train_importance.npz as dicts: the views' frames and videos (video-major), the
    steps, the images uint8 [n, H, W, 3], the reference's dz per view, its table ids and per-view counts, and the cameras."""
    g = np.load(GOLDEN)
    out = []
    for name in g["cases"]:
        name = str(name)
        n_videos, n_frames, H, W, full, kf_step, kf_frac, frac = g[f"{name}/params"]
        n_videos, n_frames, H, W = int(n_videos), int(n_frames), int(H), int(W)
        times = g[f"{name}/times"]  # frame-major over the videos (immersive.py:140-141, 352-353)
        static = tuple(int(s) for s in g[f"{name}/static"])
        seed = int(g[f"{name}/seed"])
        images = np.concatenate([video_frames(seed * 1000 + v, n_frames, H, W, static) for v in range(n_videos)])
        keep = np.unpackbits(g[f"{name}/keep"], bitorder="little", count=n_videos * n_frames * H * W).astype(bool)
        out.append(dict(
            name=name, H=H, W=W, n_videos=n_videos, n_frames=n_frames,
            frames=[int(np.round(times[f * n_videos + v] * (n_frames - 1))) for v in range(n_videos) for f in range(n_frames)],
            view_times=[float(times[f * n_videos + v]) for v in range(n_videos) for f in range(n_frames)],
            videos=[v for v in range(n_videos) for _ in range(n_frames)],
            steps=dict(load_full_step=int(full), subsample_keyframe_step=int(kf_step), subsample_keyframe_frac=float(kf_frac),
                       subsample_frac=float(frac)),
            images=images, dz=np.repeat(g[f"{name}/dz"], n_frames, axis=0), ids=np.flatnonzero(keep).astype(np.int64),
            counts=g[f"{name}/counts"], pose=g[f"{name}/pose"], K=g[f"{name}/K"], distortion=g[f"{name}/distortion"],
            cam_id=g[f"{name}/cam_id"]))
    return out
