"""Shared plumbing of the batched evaluation drivers (SURVEY.md section 8f rank 3): batching of the reference's per-image loop
and an image source that can synthesise noise images of the recorded sizes when the dataset's image folder is not mounted
(the drivers are then a throughput instrument on the REAL proposal files' box-count distribution; accuracy needs the images)."""
from __future__ import annotations

import os
import zlib
import time
from typing import Callable, Iterable, List, Optional, Sequence, Tuple

import numpy as np
from PIL import Image


# the drivers prepare (and hold on the device) this many batches of inputs at a time, and run each window through the decode slots
WINDOW = 8


def batches(items: Sequence, n: int) -> Iterable[Sequence]:
    for i in range(0, len(items), n):
        yield items[i:i + n]


class ImageSource:
    """``path(name, size_hint)`` -> a path ``vlm_fo1.mm_utils.load_image`` can open.  Real files are used when present; with
    ``synthetic_dir`` set, missing files are replaced by seeded uint8 noise of ``size_hint`` (width, height), written once."""

    def __init__(self, folder: str, synthetic_dir: Optional[str] = None):
        self.folder, self.synthetic_dir = folder, synthetic_dir
        if synthetic_dir:
            os.makedirs(synthetic_dir, exist_ok=True)

    def path(self, name: str, size_hint: Tuple[int, int]) -> str:
        real = os.path.join(self.folder, name)
        if os.path.exists(real) or not self.synthetic_dir:
            return real
        out = os.path.join(self.synthetic_dir, os.path.splitext(os.path.basename(name))[0] + ".png")
        if not os.path.exists(out):
            w, h = max(int(size_hint[0]), 28), max(int(size_hint[1]), 28)
            rng = np.random.default_rng(zlib.crc32(name.encode()))      # NOT hash(): str hashes are salted per process
            Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(out)
        return out


def size_from_boxes(boxes: Sequence[Sequence[float]], default: Tuple[int, int] = (640, 480)) -> Tuple[int, int]:
    """(width, height) that contains every proposal (for files that do not record the image size)."""
    if not boxes:
        return default
    b = np.asarray(boxes, dtype=np.float64)
    return int(np.ceil(b[:, 2].max())) + 1, int(np.ceil(b[:, 3].max())) + 1


class Throughput:
    def __init__(self) -> None:
        self.t0 = time.perf_counter(); self.n = 0

    def add(self, k: int) -> None:
        self.n += k

    def report(self, what: str) -> float:
        dt = time.perf_counter() - self.t0
        ips = self.n / dt if dt > 0 else 0.0
        print(f"{what}: {self.n} images in {dt:.1f} s = {ips:.2f} images/s")
        return ips
