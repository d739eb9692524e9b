"""mdc_jpeg_encode_device (csrc/mdc_jpeg_encode.cu) on the GPU: cv2.imencode('.jpg')'s bytes for every corpus frame, in batches of 1, 7
and 300 frames; exact sizes; padded rows never read; the same bytes on every run; argument errors refused before any launch; and a
golden fixture of OpenCV's bytes for machines without cv2."""
import ctypes as C
import os

import numpy as np
import pytest

import jpeg_encode_spec as E

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from mono_dataset_code_b200 import api  # noqa: E402
from mono_dataset_code_b200._lib import lib  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "jpeg_encode", "jpeg_encode.npz")


@pytest.fixture(scope="module")
def ctx():
    return api.Context(None, None, 0)


def imencode(img, q):
    cv2 = pytest.importorskip("cv2")
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


def encode_batch(ctx, imgs, q, pitch=None, fill=0):
    h, w = imgs[0].shape
    p = pitch or w
    buf = np.full((len(imgs), h, p), fill, np.uint8)
    for i, im in enumerate(imgs):
        buf[i, :, :w] = im
    d = torch.from_numpy(buf).cuda()
    return api.jpeg_encode_device(d[:, :, :w], q, ctx=ctx)


@pytest.mark.parametrize("w,h", E.SIZES, ids=[f"{w}x{h}" for (w, h) in E.SIZES])
def test_equals_opencv_on_the_corpus(ctx, w, h):
    cases = E.corpus(sizes=[(w, h)])
    for q in sorted({q for (_, _, q) in cases}):
        names = [n for (n, _, qq) in cases if qq == q]
        imgs = [im for (_, im, qq) in cases if qq == q]
        got = encode_batch(ctx, imgs, q)
        for name, im, g in zip(names, imgs, got):
            assert g == imencode(im, q), name


@pytest.mark.parametrize("n", [1, 7, 300])
def test_batches_equal_opencv_and_sizes_are_exact(ctx, n):
    w, h = 333, 217
    kinds = E.KINDS
    imgs = [E.frame(kinds[i % len(kinds)], w, h, seed=i) for i in range(n)]
    got = encode_batch(ctx, imgs, 95)
    assert len(got) == n
    for i, (im, g) in enumerate(zip(imgs, got)):
        assert g == imencode(im, 95), i
    # sizes_host straight from the C call
    d = torch.from_numpy(np.stack(imgs)).cuda()
    stride = api.jpeg_encode_bound(w, h)
    out = torch.empty((n, stride), dtype=torch.uint8, device="cuda")
    sizes = (C.c_size_t * n)()
    assert lib.mdc_jpeg_encode_device(ctx._h, C.c_void_p(d.data_ptr()), w, n, w, h, 95, C.c_void_p(out.data_ptr()), stride, sizes, None) == 0
    assert [sizes[i] for i in range(n)] == [len(g) for g in got]
    host = out.cpu().numpy()
    for i in range(n):
        assert host[i, :sizes[i]].tobytes() == got[i]


@pytest.mark.parametrize("fill", [0xA5, 0x00])
def test_row_padding_is_never_read(ctx, fill):
    for (w, h) in [(9, 1), (17, 23), (333, 217)]:
        imgs = [E.frame(k, w, h) for k in ("noise", "blurred", "full")]
        for q in (50, 100):
            plain = encode_batch(ctx, imgs, q)
            padded = encode_batch(ctx, imgs, q, pitch=w + 29, fill=fill)
            assert plain == padded, (w, h, q)
            assert padded == [imencode(im, q) for im in imgs]


def test_two_runs_give_identical_output(ctx):
    imgs = [E.frame(k, 640, 480, seed=s) for s in range(4) for k in ("noise", "ffbytes", "blurred")]
    a = encode_batch(ctx, imgs, 95)
    b = encode_batch(ctx, imgs, 95)
    assert a == b


def test_argument_errors_launch_nothing(ctx):
    w, h = 64, 48
    d = torch.zeros((2, h, w), dtype=torch.uint8, device="cuda")
    stride = api.jpeg_encode_bound(w, h)
    out = torch.empty((2, stride), dtype=torch.uint8, device="cuda")
    sizes = (C.c_size_t * 2)()
    F, O = C.c_void_p(d.data_ptr()), C.c_void_p(out.data_ptr())
    good = dict(c=ctx._h, f=F, pitch=w, n=2, w=w, h=h, q=95, out=O, stride=stride, sizes=sizes)

    def call(**kw):
        a = {**good, **kw}
        return lib.mdc_jpeg_encode_device(a["c"], a["f"], a["pitch"], a["n"], a["w"], a["h"], a["q"], a["out"], a["stride"], a["sizes"], None)

    before = ctx.launch_count
    bad = [dict(q=0), dict(q=101), dict(q=-5), dict(w=0), dict(h=0), dict(w=-1), dict(w=65536, pitch=70000), dict(pitch=w - 1),
           dict(stride=stride - 1), dict(f=None), dict(out=None), dict(sizes=None), dict(n=-1), dict(c=None)]
    for kw in bad:
        assert call(**kw) == 1, kw
    assert ctx.launch_count == before
    assert call(n=0, f=None, out=None, sizes=None) == 0
    assert ctx.launch_count == before
    assert lib.mdc_jpeg_encode_bound(0, 5) == 0 and lib.mdc_jpeg_encode_bound(w, h) == E.encode_bound(w, h)
    assert call() == 0
    assert ctx.launch_count == before + 5


def test_golden_fixture(ctx):
    g = np.load(GOLDEN)
    for i in range(int(g["n"])):
        img, q = g[f"img{i}"], int(g[f"q{i}"])
        got = encode_batch(ctx, [img], q)[0]
        assert got == g[f"jpg{i}"].tobytes(), i
        assert got == E.encode(img, q), i
