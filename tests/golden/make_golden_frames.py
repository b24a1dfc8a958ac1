"""Generates tests/golden/tiny_frames.npz: seeded BGR frames and depth at an odd size (161 x 121), their blur scores, the keyframe selection
over windows of 2 (3 frames: one full window and a short one), and intensity / depth levels 0-2 from tests/frames_ref.py.  The inputs are
stored so that the fixture does not depend on the generator.   Run:  python tests/golden/make_golden_frames.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

WINDOW = 2


def make_inputs(F=3, W=161, H=121, seed=11):
    """Smooth seeded colour patterns with noise, every second frame box-blurred; smooth depth with holes (zeros)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    bgr = np.empty((F, H, W, 3), np.uint8)
    for f in range(F):
        for c in range(3):
            ph = rng.uniform(0, 2 * np.pi, 2)
            v = 128 + 60 * np.sin(xx / (7 + 3 * c) + ph[0]) * np.cos(yy / (9 + 2 * f) + ph[1]) + rng.integers(-6, 7, (H, W))
            if f % 2:
                k = np.ones(5) / 5
                v = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 1, v)
                v = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 0, v)
            bgr[f, :, :, c] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    depth = np.stack([1.0 + 0.2 * np.sin(xx / 23 + f) + 0.001 * (xx // 8) for f in range(F)]).astype(np.float32)
    depth[rng.random((F, H, W)) < 0.3] = 0.0
    return bgr, depth


def main():
    import frames_ref as R
    from intrinsic3d_b200.keyframes import select_keyframes
    bgr, depth = make_inputs()
    scores = R.blur_scores(bgr)
    L, D = R.pyramid(bgr, depth, 3)
    np.savez_compressed(os.path.join(HERE, "tiny_frames.npz"), bgr=bgr, depth=depth, scores=scores, window=np.int32(WINDOW),
                        selection=select_keyframes(scores, WINDOW), lum0=L[0], lum1=L[1], lum2=L[2], depth1=D[1], depth2=D[2])
    print(f"tiny_frames.npz: {len(bgr)} frames of {bgr.shape[2]}x{bgr.shape[1]}, scores {scores}")


if __name__ == "__main__":
    main()
