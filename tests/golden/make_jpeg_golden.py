"""Writes tests/golden/jpeg_cv2.npz from cv2.imencode (diff_retrieval.py:513-515):  python tests/golden/make_jpeg_golden.py

The images are oracle.complexity.golden_images (seeded numpy), so a machine without cv2 rebuilds them exactly; only the
encodings come from cv2.  For every size, kind and quality the file holds the encoded size and its sha256; the full
bytes of the 16 x 16 and 32 x 48 noise encodings are kept as well.
  sizes   int64 [n_sizes, n_kinds, n_qualities]
  sha256  uint8 [n_sizes, n_kinds, n_qualities, 32]
  full_<h>x<w>_q<q>   uint8 bytes of the noise image's file
  qualities, hw, kinds, cv2_version
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def main():
    import cv2
    from oracle import complexity as oc
    sizes, shas, full, kinds = [], [], {}, None
    for h, w in oc.GOLDEN_SIZES:
        imgs = oc.golden_images(h, w)
        kinds = [k for k, _ in imgs]
        s_row, h_row = [], []
        for kind, img in imgs:
            s_q, h_q = [], []
            for q in oc.GOLDEN_QUALITIES:
                ok, enc = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_QUALITY), q])
                assert ok
                b = enc.tobytes()
                s_q.append(len(b))
                h_q.append(np.frombuffer(hashlib.sha256(b).digest(), np.uint8))
                if kind == "noise" and h * w <= 32 * 48:
                    full[f"full_{h}x{w}_q{q}"] = np.frombuffer(b, np.uint8)
            s_row.append(s_q)
            h_row.append(h_q)
        sizes.append(s_row)
        shas.append(h_row)
    np.savez_compressed(os.path.join(HERE, "jpeg_cv2.npz"), sizes=np.array(sizes, np.int64),
                        sha256=np.array(shas, np.uint8), qualities=np.array(oc.GOLDEN_QUALITIES),
                        hw=np.array(oc.GOLDEN_SIZES), kinds=np.array(kinds), cv2_version=np.array(cv2.__version__),
                        **full)


if __name__ == "__main__":
    main()
