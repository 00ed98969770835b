"""The JPEG corpus of tests/golden/jpeg_corpus.npz (made by tests/golden/make_golden_jpeg.py) as Python objects.

Every supported file carries the SHA-256 of Pillow's planar decode; the dataset faces also carry the decode itself."""
import hashlib
import os

import numpy as np

CORPUS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_corpus.npz")


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


class Entry:
    def __init__(self, z, i):
        self.name = str(z["names"][i])
        self.bytes = z["data"][z["offsets"][i]:z["offsets"][i + 1]].tobytes()
        self.C, self.H, self.W = int(z["C"][i]), int(z["H"][i]), int(z["W"][i])
        self.info_rc, self.upload_rc = int(z["info_rc"][i]), int(z["upload_rc"][i])
        self.cache_hw = (int(z["cache_h"][i]), int(z["cache_w"][i]))
        self.face = bool(z["faces"][i])
        self.sha256 = str(z["sha256"][i])
        d = z["decoded"][z["dec_offsets"][i]:z["dec_offsets"][i + 1]]
        self.decoded = d.reshape(self.C, self.H, self.W) if d.size else None

    @property
    def supported(self):
        return self.upload_rc == 0

    def expected(self, Cs):
        """Pillow's decode as image.load(path, Cs, 'byte') gives it (a 1-component file replicated under Cs = 3);
        stored for the dataset faces only."""
        assert self.decoded is not None, "%s: only the SHA-256 of its decode is stored" % self.name
        return np.repeat(self.decoded, 3, axis=0) if Cs == 3 and self.C == 1 else self.decoded

    def mismatch(self, got):
        """None when a cache row `got` [Cs][H][W] is Pillow's decode bit for bit (a 1-component file replicated to
        every plane), else what differs."""
        got = np.asarray(got)
        if got.shape[1:] != (self.H, self.W) or got.shape[0] not in (self.C, 3):
            return "shape %s, expected [%s][%d][%d]" % (got.shape, "1 or 3" if self.C == 1 else 3, self.H, self.W)
        if self.C == 1 and got.shape[0] == 3 and not (np.array_equal(got[0], got[1]) and np.array_equal(got[0], got[2])):
            return "the planes of a 1-component file differ"
        h = digest(got[:self.C])
        return None if h == self.sha256 else "SHA-256 %s, Pillow's decode has %s" % (h[:16], self.sha256[:16])


def load():
    with np.load(CORPUS) as z:
        return [Entry(z, i) for i in range(len(z["names"]))]
