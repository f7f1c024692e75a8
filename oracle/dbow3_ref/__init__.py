"""The compiled, unmodified DBoW3 of the reference (built by build.py into oracle/_ref/) behind the small surface
DBoW3Py gives vista_slam/loop_detector.py: load, transform, score."""
import ctypes

import numpy as np

from oracle import loop_detector_oracle as O


class RefVocabulary:
    """The compiled, unmodified DBoW3 (oracle/dbow3_ref) behind the small surface DBoW3Py gives loop_detector.py."""

    def __init__(self, lib, handle=None):
        self.L, self.h = lib, handle

    def load(self, path):
        err = ctypes.create_string_buffer(512)
        self.h = self.L.dbow_load(path.encode(), err, 512)
        if not self.h:
            raise RuntimeError(err.value.decode())

    def transform(self, desc):
        d = np.ascontiguousarray(desc, np.uint8)
        cap = max(len(d), 1)
        w, v = np.zeros(cap, np.int32), np.zeros(cap, np.float64)
        n = self.L.dbow_transform(self.h, d.ctypes.data, len(d), w.ctypes.data, v.ctypes.data, cap)
        return w[:n].astype(np.int64), v[:n]

    def score(self, a, b):
        wa, va = np.ascontiguousarray(a[0], np.int32), np.ascontiguousarray(a[1], np.float64)
        wb, vb = np.ascontiguousarray(b[0], np.int32), np.ascontiguousarray(b[1], np.float64)
        return self.L.dbow_score(self.h, wa.ctypes.data, va.ctypes.data, len(wa), wb.ctypes.data, vb.ctypes.data,
                                 len(wb))

    def tree(self):
        """The loaded tree as an oracle Vocabulary (node ids as DBoW3 holds them)."""
        n = self.L.dbow_nodes(self.h)
        info = np.zeros(4, np.int32)
        parent, word = np.zeros(n, np.int32), np.zeros(n, np.int32)
        weight, desc = np.zeros(n, np.float64), np.zeros((n, 32), np.uint8)
        ch = np.zeros((max(n - 1, 1), 2), np.int32)
        m = self.L.dbow_dump(self.h, info.ctypes.data, parent.ctypes.data, weight.ctypes.data, desc.ctypes.data,
                             word.ctypes.data, ch.ctypes.data)
        v = O.Vocabulary(int(info[0]), int(info[1]), int(info[2]), int(info[3]), parent, desc, weight, word)
        for p, c in ch[:m]:
            v.children[p].append(int(c))
        return v
