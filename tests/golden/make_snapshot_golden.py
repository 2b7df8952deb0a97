"""Writes tests/golden/reference/snapshot_*.npz with the reference's own build_super_images /
build_super_shape_images / drawCaption (imported read-only from /root/reference, so this script only works where the
reference is).  skimage is absent: its pyramid_expand is the restatement in oracle/snapshot_oracle.py (rules and
version in its docstring).  The font is Pillow's built-in one at size 50 in place of the dataset's FreeMono.  The
inputs are rebuilt from seeds (tests/snapshot_cases.py); each file holds the canvas rows of the first ``keep``
images and the inputs' checksum.

    python tests/golden/make_snapshot_golden.py
"""
import os
import sys

import numpy as np
from PIL import ImageFont

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import refimport  # noqa: E402
import snapshot_cases as C  # noqa: E402
from oracle import snapshot_oracle as O  # noqa: E402


def main():
    ref = refimport.load(18)
    sys.modules["skimage.transform"].pyramid_expand = O.pyramid_expand
    font = ImageFont.load_default(size=50)
    ImageFont.truetype = lambda *a, **k: font
    out = os.path.join(HERE, "reference")
    for name, c in C.CASES.items():
        imgs, lr, maps, lens, caps = C.inputs(name)
        with np.errstate(all="ignore"):
            if c.get("shape"):
                canvas, _ = ref.utils.build_super_shape_images(imgs, caps, C.IXTOWORD, maps, c["att"], font_max=20,
                                                               font_size=12, max_word_num=c["words"],
                                                               batch_size=c["b"])
            else:
                per = [maps[i:i + 1, :int(lens[i])] for i in range(c["b"])] if lens is not None else maps
                canvas, _ = ref.utils.build_super_images(imgs, caps, C.IXTOWORD, per, c["att"], lr_imgs=lr,
                                                         max_word_num=c["words"])
        path = os.path.join(out, "snapshot_%s.npz" % name)
        np.savez_compressed(path, canvas=canvas[:C.rows(name)], checksum=C.checksum(name))
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
