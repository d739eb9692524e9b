"""The plain-C restatement of responseCalib's plotE / plotG (tests/cpp/rc_plot_oracle.c), built as the reference is built (-O3, no
contraction, the flags of oracle/Makefile's `port` target) against the host's libm, and loaded with ctypes; the host libm's exp and
log through the same library; and the reference program's raw imwrite dumps (MDC_SHIM_DUMP_DIR).  The restatement is kept with the
tests rather than in oracle/port so that the oracle the existing tests pin stays exactly as it is."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import jpeg_encode_spec as JS

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        with tempfile.TemporaryDirectory(prefix="rc_plot_oracle_") as d:      # the loaded library outlives its file
            so = os.path.join(d, "librc_plot_oracle.so")
            subprocess.run(["gcc", "-O3", "-std=c99", "-ffp-contract=off", "-fPIC", "-shared", os.path.join(HERE, "cpp", "rc_plot_oracle.c"),
                            "-o", so, "-lm"], check=True)
            lib_ = C.CDLL(so)
        vp = C.c_void_p
        for name, args in (("oport_rc_plot_e_range", [vp, C.c_int, vp]), ("oport_rc_plot_e_map", [vp, C.c_int, vp, vp, vp]),
                           ("oport_rc_plot_g", [vp, vp, vp]), ("oport_libm", [C.c_int, vp, vp, C.c_size_t])):
            getattr(lib_, name).argtypes = args
            getattr(lib_, name).restype = None
        _lib = lib_
    return _lib


def libm(x, op):
    """exp or log (op "exp" / "log") of the host's libm, as the reference program calls them"""
    x = np.ascontiguousarray(x, np.float64)
    out = np.empty_like(x)
    lib().oport_libm(0 if op == "exp" else 1, x.ctypes.data, out.ctypes.data, x.size)
    return out


def plot_e_range(E):
    E = np.ascontiguousarray(E, np.float64).reshape(-1)
    r = np.empty(4)
    lib().oport_rc_plot_e_range(E.ctypes.data, E.size, r.ctypes.data)
    return r


def plot_e_map(E, range4):
    """-> (bgr uint8 [npix, 3], e16 uint16 [npix])"""
    E = np.ascontiguousarray(E, np.float64).reshape(-1)
    range4 = np.ascontiguousarray(range4, np.float64)
    bgr, e16 = np.empty((E.size, 3), np.uint8), np.empty(E.size, np.uint16)
    lib().oport_rc_plot_e_map(E.ctypes.data, E.size, range4.ctypes.data, bgr.ctypes.data, e16.ctypes.data)
    return bgr, e16


def plot_e(E):
    """plotE: (bgr uint8 [npix, 3] in BGR order, e16 uint16 [npix], range {min ln(E+20), max ln(E+20), min E, max E})"""
    r = plot_e_range(E)
    return (*plot_e_map(E, r), r)


def plot_g_float(G):
    """plotG: (GImg * 255 as float32 [256, 256], the Mat handed to cv::imwrite; (min G, max G))"""
    G = np.ascontiguousarray(G, np.float64)
    out, mm = np.empty((256, 256), np.float32), np.empty(2)
    lib().oport_rc_plot_g(G.ctypes.data, out.ctypes.data, mm.ctypes.data)
    return out, (mm[0], mm[1])


def plot_g(G):
    """plotG as G-k.png holds it: the float image converted to 8 bits as cv::imwrite converts it; (min G, max G)"""
    f, mm = plot_g_float(G)
    return JS.conv_u8(f), mm


def read_dump(path):
    """A Mat the reference program handed to cv::imwrite: (rows, cols, type, pixels as a numpy array of the Mat's element type)"""
    raw = np.fromfile(path, dtype=np.uint8)
    rows, cols, typ = (int(v) for v in np.frombuffer(raw[:12].tobytes(), dtype=np.int32))
    dtype = {0: np.uint8, 16: np.uint8, 2: np.uint16, 5: np.float32}[typ]
    return rows, cols, typ, raw[12:].view(dtype)
