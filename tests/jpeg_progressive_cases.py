"""Inputs for the progressive JPEG tests: the size x channels x quality x content matrix, all generated from seeds."""
import numpy as np

SIZES = [(1, 1), (7, 5), (8, 8), (15, 17), (16, 16), (33, 47), (255, 257), (256, 256), (1920, 1080)]
CHANNELS = [1, 3, 4]
QUALITIES = [1, 10, 50, 75, 85, 95, 100]
CONTENTS = ["noise", "gradient", "edges"]


def image(content: str, w: int, h: int, ch: int, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed + 7919 * w + 104729 * h + ch)
    shape = (h, w, ch) if ch > 1 else (h, w)
    if content == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if content == "gradient":  # smooth: most AC coefficients quantise to zero, long EOB runs
        y = np.linspace(0, 1, h, dtype=np.float32)[:, None]
        x = np.linspace(0, 1, w, dtype=np.float32)[None, :]
        planes = [(255 * (0.2 + 0.6 * (a * x + (1 - a) * y))) for a in np.linspace(0.2, 0.8, max(ch, 1))]
        img = np.stack([np.broadcast_to(p, (h, w)) for p in planes], axis=-1).round().astype(np.uint8)
        return img if ch > 1 else img[..., 0]
    if content == "edges":  # sparse: a flat field with a few sharp lines and boxes
        img = np.full(shape, 40, dtype=np.uint8)
        for _ in range(4):
            x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
            img[y0:y0 + max(1, h // 7), x0:x0 + 1] = 230
            img[y0:y0 + 1, x0:x0 + max(1, w // 5)] = 200
            img[y0:y0 + 3, x0:x0 + 3] = rng.integers(0, 256)
        return img
    if content == "flat":
        return np.full(shape, 128, dtype=np.uint8)
    raise ValueError(content)


def matrix():
    """(content, w, h, ch, q): every size x channels x quality, the three contents in turn, plus flat 2048x2048.
    The 1080p cases keep one quality per content so the matrix stays a few seconds long."""
    out = []
    for w, h in SIZES:
        for ch in CHANNELS:
            for i, q in enumerate(QUALITIES):
                for j, content in enumerate(CONTENTS):
                    if (w, h) == (1920, 1080) and (i + ch) % len(QUALITIES) != 3 * j % len(QUALITIES):
                        continue
                    out.append((content, w, h, ch, q))
    for ch in CHANNELS:
        for q in (50, 100):
            out.append(("flat", 2048, 2048, ch, q))
    return out
