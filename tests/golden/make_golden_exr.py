"""Write the OpenEXR fixtures of tests/test_exr.py with OpenCV's codec (an independent writer of the format):

    OPENCV_IO_ENABLE_OPENEXR=1 python tests/golden/make_golden_exr.py

exr/<compression>_<type>_<channels>.exr for the compressions NONE, RLE, ZIPS, ZIP and PIZ (the last one must be
refused), pixel types FLOAT and HALF, and one channel (Y) or three (B, G, R: the reader takes R).  The pixels are
fixture_values(): a 13 x 7 ramp with a constant block, so that RLE finds runs, and zfar-like large values."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def fixture_values():
    a = (np.arange(13 * 7, dtype=np.float32).reshape(13, 7) * np.float32(0.37) + np.float32(0.5))
    a[4:9, 1:6] = 100.0
    return a


def main():
    os.environ.setdefault("OPENCV_IO_ENABLE_OPENEXR", "1")
    import cv2
    a = fixture_values()
    out = os.path.join(HERE, "exr")
    os.makedirs(out, exist_ok=True)
    comps = {"none": cv2.IMWRITE_EXR_COMPRESSION_NO, "rle": cv2.IMWRITE_EXR_COMPRESSION_RLE,
             "zips": cv2.IMWRITE_EXR_COMPRESSION_ZIPS, "zip": cv2.IMWRITE_EXR_COMPRESSION_ZIP,
             "piz": cv2.IMWRITE_EXR_COMPRESSION_PIZ}
    types = {"float": cv2.IMWRITE_EXR_TYPE_FLOAT, "half": cv2.IMWRITE_EXR_TYPE_HALF}
    for cn, cc in comps.items():
        for tn, tc in types.items():
            for ch, img in ((1, a), (3, np.stack([a * 2, a * 3, a], -1))):   # BGR: R = a
                if cn == "piz" and (tn, ch) != ("float", 1):
                    continue
                path = os.path.join(out, "%s_%s_%d.exr" % (cn, tn, ch))
                assert cv2.imwrite(path, img, [cv2.IMWRITE_EXR_COMPRESSION, cc, cv2.IMWRITE_EXR_TYPE, tc])


if __name__ == "__main__":
    main()
