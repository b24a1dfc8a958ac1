"""Keyframe selection on the host: the window rule and the keyframes file of the reference's KeyframeSelection
(src/keyframe_selection.cpp:73-106, 139-207).  The per-frame blur scores come from Engine.keyframe_scores (on the device)."""
from __future__ import annotations

import math
import re

import numpy as np


def select_keyframes(scores, window: int) -> np.ndarray:
    """KeyframeSelection::selectKeyframes: ceil(n / window) windows of `window` frames (the last one may be short); in each, the frame with
    the largest score wins on a strict `>` against a running maximum that starts at 0.0, so ties go to the earlier frame and a window whose
    scores are all <= 0 or NaN keeps its first frame.  Returns a bool array [n]."""
    window = int(window)
    if window <= 0:
        raise ValueError(f"select_keyframes: window must be > 0 (got {window})")
    s = [float(x) for x in np.asarray(scores, np.float64).ravel()]
    n = len(s)
    keep = np.zeros(n, bool)
    for beg in range(0, n, window):
        best, arg = 0.0, beg
        for i in range(beg, min(beg + window, n)):
            if s[i] > best:
                best, arg = s[i], i
        keep[arg] = True
    return keep


def save_keyframes(path, scores, is_keyframe, window: int) -> None:
    """KeyframeSelection::save: the window size on the first line, then one "%.6f %d" line (score, keyframe flag) per frame."""
    scores = np.asarray(scores, np.float64).ravel()
    flags = np.asarray(is_keyframe, bool).ravel()
    if len(scores) == 0 or len(scores) != len(flags):
        raise ValueError("save_keyframes: need one flag per score and at least one frame")
    with open(path, "w") as f:
        f.write(f"{int(window)}\n")
        for sc, kf in zip(scores, flags):
            f.write(f"{_fixed6(sc)} {int(kf)}\n")


def _fixed6(x: float) -> str:
    # std::fixed << setprecision(6) prints non-finite values as nan / inf / -inf
    if math.isnan(x):
        return "-nan" if math.copysign(1.0, x) < 0 else "nan"
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    return f"{x:.6f}"


_NUM = re.compile(r"[+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?")
_INT = re.compile(r"[+-]?\d+")


def load_keyframes(path):
    """KeyframeSelection::load: returns (window, scores float64 [n], is_keyframe bool [n]).  Empty lines are skipped; reading stops at the
    first line whose score or flag does not parse, as `iss >> score >> is_kf` does (`nan` is not a number to it, and a flag is 0 or 1), so
    a saved `nan` score truncates the list there.  Raises ValueError when the first line holds no window size."""
    with open(path) as f:
        lines = f.read().split("\n")
    m = _INT.match(lines[0].lstrip()) if lines else None
    if m is None:
        raise ValueError(f"load_keyframes: {path}: no window size on the first line")
    window = int(m.group())
    scores, flags = [], []
    for line in lines[1:]:
        if not line:
            continue
        tok = line.split()
        if len(tok) < 2 or not _NUM.fullmatch(tok[0]):
            break
        k = _INT.match(tok[1])
        if k is None or int(k.group()) not in (0, 1):
            break
        scores.append(float(tok[0]))
        flags.append(int(k.group()) == 1)
    return window, np.array(scores, np.float64), np.array(flags, bool)
