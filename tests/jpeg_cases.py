"""JPEG inputs shared by the CPU test of the GPU decoder's core (test_jpeg_entropy_host.py) and its GPU tests (test_jpeg_decode_gpu.py):
the corpus of test_jpeg_decoder.py, scans cut at seeded byte offsets, and seeded damage in the four modes of tests/cpp/decoder_fuzz.cpp."""
import numpy as np

from test_jpeg_decoder import CASES, scene

cv2 = __import__("cv2")

GREY_SIZES = [(64, 48), (83, 61), (8, 8), (1, 1), (17, 129), (640, 480)]
SAMPLINGS = ("444", "422", "420", "411", "440")


def corpus():
    """(w, h, bytes) of every file test_jpeg_decoder.py decodes: grey at six sizes x four scenes x qualities 35/90/100 x
    (plain, optimised tables, restart interval 3); colour in every sampling mode; the seeded random sweep."""
    out = []
    for (w, h) in GREY_SIZES:
        rng = np.random.default_rng(w * 1000 + h)
        for kind, quality in CASES:
            img = scene(rng, h, w, kind)
            for extra in ([], [cv2.IMWRITE_JPEG_OPTIMIZE, 1], [cv2.IMWRITE_JPEG_RST_INTERVAL, 3]):
                ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, quality] + extra)
                out.append((w, h, enc.tobytes()))
    if hasattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR"):
        rng = np.random.default_rng(5)
        for sampling in SAMPLINGS:
            factor = getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + sampling)
            for (w, h) in ((96, 64), (75, 53), (33, 17)):
                bgr = np.stack([scene(rng, h, w, k) for k in ("smooth", "noise", "ramp")], axis=-1)
                for quality in (50, 95):
                    for extra in ([], [cv2.IMWRITE_JPEG_RST_INTERVAL, 2]):
                        ok, enc = cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, factor] + extra)
                        out.append((w, h, enc.tobytes()))
    rng = np.random.default_rng(2024)
    factors = [getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + s) for s in SAMPLINGS] if hasattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR") else []
    for _ in range(60):
        w, h = int(rng.integers(1, 200)), int(rng.integers(1, 160))
        img = scene(rng, h, w, ("smooth", "noise", "edges", "ramp")[int(rng.integers(0, 4))])
        params = [cv2.IMWRITE_JPEG_QUALITY, int(rng.integers(1, 101))]
        if rng.random() < 0.3:
            params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
        if rng.random() < 0.3:
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, int(rng.integers(1, 9))]
        if factors and rng.random() < 0.5:
            img = np.stack([img, np.roll(img, 3, 1), 255 - img], axis=2)
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, factors[int(rng.integers(0, len(factors)))]]
        ok, enc = cv2.imencode(".jpg", img, params)
        out.append((w, h, enc.tobytes()))
    return out


def scan_start(blob):
    """Offset of the first entropy-coded byte (after the SOS segment)."""
    at = blob.find(b"\xff\xda")
    return at + 2 + ((blob[at + 2] << 8) | blob[at + 3])


def scan_cuts(files, per_file=3, seed=31):
    """Files truncated at seeded offsets inside their scan: the decoder reads zero bits from the cut on."""
    rng = np.random.default_rng(seed)
    out = []
    for (w, h, blob) in files:
        s = scan_start(blob)
        if len(blob) - s < 8:
            continue
        for _ in range(per_file):
            out.append((w, h, blob[: int(rng.integers(s + 1, len(blob) - 2))]))
    return out


def fuzz_bases():
    """The two JPEGs tests/test_decoder_fuzz.py damages: grey quality 85, and colour quality 60 with restart interval 4 (200 x 120)."""
    rng = np.random.default_rng(3)
    yy, xx = np.mgrid[0:120, 0:200]
    img = np.clip(40 + 0.6 * xx + rng.normal(0, 12, (120, 200)), 0, 255).astype(np.uint8)
    grey = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 85])[1].tobytes()
    colour = cv2.imencode(".jpg", np.stack([img, 255 - img, img], 2), [cv2.IMWRITE_JPEG_QUALITY, 60, cv2.IMWRITE_JPEG_RST_INTERVAL, 4])[1].tobytes()
    return {"grey": grey, "colour_rst": colour}


def damaged(base, rounds, seed):
    """decoder_fuzz.cpp's damage, seeded: round r % 4 = 0 random bytes anywhere, 1 random bytes in the first 700 (headers and
    tables), 2 truncation, 3 a run of 0xFF."""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(rounds):
        b = bytearray(base)
        mode = r % 4
        if mode == 0:
            for _ in range(1 + int(rng.integers(0, 8))):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
        elif mode == 1:
            for _ in range(1 + int(rng.integers(0, 4))):
                b[int(rng.integers(0, min(len(b), 700)))] = int(rng.integers(0, 256))
        elif mode == 2:
            b = b[: int(rng.integers(0, len(b)))]
        else:
            p = int(rng.integers(0, len(b)))
            n = min(len(b) - p, 1 + int(rng.integers(0, 64)))
            b[p:p + n] = b"\xff" * n
        out.append(bytes(b))
    return out


def damaged_set(rounds=1500):
    """The damaged files the CPU sanitizer test checks; the GPU test decodes the same set."""
    return [(name, blob) for i, (name, base) in enumerate(sorted(fuzz_bases().items())) for blob in damaged(base, rounds, 100 + i)]
