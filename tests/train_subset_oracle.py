"""NumPy restatement of the training table of ``hr_sample_train_rows`` (csrc/hr_train_batch.cu): the video datasets'
per-frame pixel subsets, the table order, the rank -> pixel map and the draws with replacement.

* ``plan``: one ``(stride, offset)`` per view, with the reference's two counter conventions (technicolor.py:211-236,
  neural_3d.py:168-185,217-269), written as the reference's loops are.
* ``table``: the pixel ids ``view*H*W + y*W + x`` of the whole table by masking, views in order and ``np.nonzero`` order
  within a view (the reference's ``coords[mask]``).
* ``rank_to_pixel``: the kernel's closed form, vectorised.
* ``draws``: row ``i = b*B + r`` of epoch ``e`` is ``umulhi(mix64(draw_key + G*(i + 1)), n)``,
  ``draw_key = mix64(mix64(seed ^ DRAW_DOMAIN) + G*(e + 1))``.
"""
import numpy as np

from tests.train_order_oracle import GOLDEN, M64, mix64, mix64_int

DRAW_DOMAIN = 0x5245504C41434531


def plan(frames, load_full_step, subsample_keyframe_step, subsample_keyframe_frac, subsample_frac, counters, videos=None):
    kf_every = int(np.round(1.0 / subsample_keyframe_frac))
    fr_every = int(np.round(1.0 / subsample_frac))
    out = []
    keyframe_offset = frame_offset = 0
    for i, frame in enumerate(frames):
        if counters == "neural_3d" and (i == 0 or videos[i] != videos[i - 1]):
            keyframe_offset = frame_offset = videos[i]  # neural_3d.py:224-226, and frame_idx == 0 is whole (:262-263)
            out.append((1, 0))
        elif frame % load_full_step == 0:
            out.append((1, 0))
        elif frame % subsample_keyframe_step == 0:
            out.append((kf_every, keyframe_offset))
            keyframe_offset += 1
        else:
            out.append((fr_every, frame_offset))
            frame_offset += 1
    return out


def mask(stride, offset, H, W):
    y, x = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return (x + y + offset) % stride == 0


def table(rules, H, W):
    return np.concatenate([v * H * W + np.nonzero(mask(s, o, H, W).reshape(-1))[0] for v, (s, o) in enumerate(rules)])


def counts(rules, H, W):
    return np.array([int(mask(s, o, H, W).sum()) for s, o in rules], dtype=np.int64)


def rank_to_pixel(stride, offset, H, W, q):
    """(y, x) of rank ``q`` of a view's kept pixels: the block of ``stride`` rows holding it, then a walk over those rows."""
    q = np.asarray(q, dtype=np.int64)
    s = stride
    y = (q // W) * s
    rem = q - (q // W) * W
    found_y, found_x = np.full(q.shape, -1), np.full(q.shape, -1)
    todo = np.ones(q.shape, dtype=bool)
    for _ in range(s):
        x0 = (s - (y + offset) % s) % s
        cnt = np.where(x0 < W, (W - 1 - x0) // s + 1, 0)
        hit = todo & (rem < cnt) & (y < H)
        found_y[hit], found_x[hit] = y[hit], (x0 + s * rem)[hit]
        todo &= ~hit
        rem = np.where(todo, rem - cnt, rem)
        y = y + 1
    return found_y, found_x


def table_pixels(rules, H, W, k):
    """The pixel ids of table rows ``k`` through the closed form."""
    k = np.asarray(k, dtype=np.int64)
    start = np.concatenate([[0], np.cumsum(counts(rules, H, W))])
    v = np.searchsorted(start, k, side="right") - 1
    out = np.empty(k.shape, dtype=np.int64)
    for view in np.unique(v):
        sel = v == view
        s, o = rules[view]
        y, x = rank_to_pixel(s, o % s, H, W, k[sel] - start[view])
        out[sel] = view * H * W + y * W + x
    return out


def _mulhi(a: np.ndarray, n: int) -> np.ndarray:
    """The high 64 bits of the 128-bit product of uint64 ``a`` and ``n`` < 2^63."""
    m32 = np.uint64(0xFFFFFFFF)
    s32 = np.uint64(32)
    a_lo, a_hi = a & m32, a >> s32
    b_lo, b_hi = np.uint64(n & 0xFFFFFFFF), np.uint64(n >> 32)
    with np.errstate(over="ignore"):
        p0, p1, p2, p3 = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
        mid = (p0 >> s32) + (p1 & m32) + (p2 & m32)
        return p3 + (p1 >> s32) + (p2 >> s32) + (mid >> s32)


def draw_key(seed: int, epoch: int) -> int:
    return mix64_int(mix64_int((seed ^ DRAW_DOMAIN) & M64) + GOLDEN * ((epoch + 1) & M64))


def draws(n: int, seed: int, epoch: int, positions) -> np.ndarray:
    """The table rows drawn at ``positions`` (``b*B + r``) of epoch ``epoch``."""
    i = np.asarray(positions, dtype=np.uint64)
    with np.errstate(over="ignore"):
        state = np.uint64(draw_key(seed, epoch)) + np.uint64(GOLDEN) * (i + np.uint64(1))
    return _mulhi(mix64(state), n).astype(np.int64)
