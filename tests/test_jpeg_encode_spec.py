"""The numpy restatement of cv::imwrite(".jpg") for single-channel images (tests/jpeg_encode_spec.py) against OpenCV itself, byte for byte:
every corpus frame at every quality, and the float path (a CV_32F image is converted with saturate_cast<uchar> first).  No GPU."""
import numpy as np
import pytest

import jpeg_encode_spec as E

cv2 = pytest.importorskip("cv2")


def imencode(img, q=None):
    params = [] if q is None else [cv2.IMWRITE_JPEG_QUALITY, q]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


@pytest.mark.parametrize("w,h", E.SIZES, ids=[f"{w}x{h}" for (w, h) in E.SIZES])
def test_spec_equals_opencv(w, h):
    for name, img, q in E.corpus(sizes=[(w, h)]):
        assert E.encode(img, q) == imencode(img, q), name


def test_header_is_328_bytes_and_quality_table_is_clamped():
    assert len(E.header(1, 1, 95)) == E.HEADER_BYTES == 328
    assert E.quant_table(1).max() == 255 and E.quant_table(100).min() == 1
    assert imencode(np.zeros((5, 5), np.uint8), 95)[:E.HEADER_BYTES] == E.header(5, 5, 95)


def test_many_stuffed_bytes_in_the_ff_frame():
    img = E.frame("ffbytes", 640, 480)
    data = E.encode(img, 95)[E.HEADER_BYTES:-2]
    assert data.count(b"\xff\x00") > 1000


def test_float_images_are_converted_like_saturate_cast():
    rng = np.random.default_rng(5)
    x = rng.uniform(-300, 600, (37, 51)).astype(np.float32)
    x.flat[::7] = np.rint(x.flat[::7]) + 0.5                               # exact half-integers: round half to even
    x.flat[1::11] = np.nan
    x.flat[2::13] = np.inf
    x.flat[3::17] = -np.inf
    x.flat[4::19] = 2.0 ** 31
    x.flat[5::23] = 3e9
    x.flat[6::29] = -2.0 ** 31 - 1e3
    x.flat[8::31] = -0.5
    u = E.conv_u8(x)
    assert imencode(x) == E.encode(u, 95)
    for q in (10, 95, 100):
        assert imencode(x, q) == E.encode(u, q)
    assert u.flat[4] == 0 and u.flat[5] == 0 and u.flat[1] == 0 and u.flat[2] == 0      # >= 2^31, NaN, inf -> 0
