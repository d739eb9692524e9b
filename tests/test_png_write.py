"""mdc_png_write (the library's PNG writer, which responseCalib_b200 and vignetteCalib_b200 write their images with): 8-bit grey,
8-bit BGR and 16-bit grey images from 1 x 1 up to odd widths, from packed and padded rows, decode with cv2.imread(IMREAD_UNCHANGED)
to the pixels that were passed in, as cv2.imwrite's own files do; bad arguments and unwritable paths are refused."""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from mono_dataset_code_b200 import api  # noqa: E402

SIZES = [(1, 1), (1, 7), (7, 1), (2, 3), (33, 17), (257, 5), (640, 480), (1001, 3)]
KINDS = {"grey8": (np.uint8, None), "bgr8": (np.uint8, 3), "grey16": (np.uint16, None)}


def image(rng, w, h, dtype, ch, pattern):
    shape = (h, w) if ch is None else (h, w, ch)
    hi = np.iinfo(dtype).max
    if pattern == "random":
        return rng.integers(0, hi + 1, shape, dtype=dtype)
    if pattern == "flat":
        return np.full(shape, hi // 3, dtype)
    x = np.arange(w)[None, :] * 37 + np.arange(h)[:, None] * 11                      # ramps that wrap, so Sub sees every difference
    return np.broadcast_to((x % (hi + 1)).astype(dtype)[..., None] if ch else (x % (hi + 1)).astype(dtype), shape).copy()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("w,h", SIZES)
def test_png_decodes_to_the_pixels_written(tmp_path, kind, w, h):
    dtype, ch = KINDS[kind]
    rng = np.random.default_rng(w * 1000 + h)
    for pattern in ("random", "flat", "ramp"):
        img = image(rng, w, h, dtype, ch, pattern)
        for pad in (0, 5):
            # rows `pad` elements wider than the image, filled with garbage that must not reach the file
            buf = rng.integers(0, np.iinfo(dtype).max, (h, w + pad) + (() if ch is None else (ch,)), dtype=dtype)
            buf[:, :w] = img
            path = str(tmp_path / f"{pattern}_{pad}.png")
            api.png_write(path, buf[:, :w])
            back = cv2.imread(path, cv2.IMREAD_UNCHANGED)
            assert back is not None and back.dtype == dtype and back.shape == img.shape, (pattern, pad)
            assert np.array_equal(back, img), (pattern, pad)
            ref = str(tmp_path / f"cv2_{pattern}_{pad}.png")
            cv2.imwrite(ref, img)
            assert np.array_equal(cv2.imread(ref, cv2.IMREAD_UNCHANGED), back)


def test_png_write_refuses_bad_arguments(tmp_path):
    from mono_dataset_code_b200._lib import lib
    img = np.zeros((4, 4), np.uint8)
    p = str(tmp_path / "x.png").encode()
    assert lib.mdc_png_write(p, img.ctypes.data, 4, 4, 4, 12, 1) == 1          # depth
    assert lib.mdc_png_write(p, img.ctypes.data, 4, 4, 4, 8, 2) == 1           # channels
    assert lib.mdc_png_write(p, img.ctypes.data, 4, 4, 3, 8, 1) == 1           # rows shorter than the image
    assert lib.mdc_png_write(p, img.ctypes.data, 0, 4, 4, 8, 1) == 1
    assert lib.mdc_png_write(p, None, 4, 4, 4, 8, 1) == 1
    assert not os.path.exists(p.decode())
    with pytest.raises(api.MdcError, match="IO"):
        api.png_write(str(tmp_path / "no_such_dir" / "x.png"), img)
