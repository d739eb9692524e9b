"""Python host-side mirror of the reference's operator interface for the hot path.

Same names, argument meaning and error behaviour as the reference's C++ classes
(/root/reference/src/FOVUndistorter.h:36-83, PhotometricUndistorter.h:37-45,
BenchmarkDatasetReader.h:83-243), implemented on the C ABI of libmdc_b200.so.  The C++ mirror
lives in include/compat/*.h; this module exists so tests and bench.py read like the
reference's call sites.  torch is used for device memory, streams and torch.distributed only.

Host arrays (numpy) go through the library's host-buffer entry points (H2D + kernel + D2H);
CUDA tensors are processed in place on the device with no copies.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import lib, check, MdcError, RECTIFY, REMOVE_GAMMA, REMOVE_VIGNETTE, NAN_OVEREXPOSED  # noqa: F401

_f32p = C.POINTER(C.c_float)


def _np_f32(ptr, n):
    return np.ctypeslib.as_array(ptr, (n,)).copy() if ptr else None


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


_OUT_TYPES = {"float32": _lib.OUT_F32, "float16": _lib.OUT_F16, "uint8": _lib.OUT_U8}


def _dtype_name(dtype) -> str:
    """'float32' / 'float16' / 'uint8' / ... for a torch or numpy dtype (None = float32)."""
    if dtype is None:
        return "float32"
    if type(dtype).__module__.startswith("torch"):
        return str(dtype).split(".")[-1]
    return np.dtype(dtype).name


def _out_type(dtype) -> int:
    """The MDC_OUT_* of a torch / numpy dtype; prepared levels come as float32 (default), float16 or uint8."""
    name = _dtype_name(dtype)
    if name not in _OUT_TYPES:
        raise ValueError(f"prepared levels are float32, float16 or uint8, not {dtype}")
    return _OUT_TYPES[name]


def _check_out_dtype(outs, dtype):
    """Caller-supplied level buffers must have the requested element type (raw integer addresses are taken as they are)."""
    want = _dtype_name(dtype)
    for i, o in enumerate(outs):
        if hasattr(o, "dtype") and _dtype_name(o.dtype) != want:
            raise ValueError(f"output level {i} is {o.dtype}, expected {want}")


def _flags(rectify, gamma, vignette, nan_over) -> int:
    return (RECTIFY if rectify else 0) | (REMOVE_GAMMA if gamma else 0) | (REMOVE_VIGNETTE if vignette else 0) | \
        (NAN_OVEREXPOSED if nan_over else 0)


class UndistorterFOV:
    """FOV-model rectifier (FOVUndistorter.h:36).  Invalid objects behave like the reference's:
    isValid() is False and undistort() leaves the output untouched."""

    def __init__(self, configFileName: str | None = None, *, float_math: bool = False, params=None):
        h = C.c_void_p()
        self.status = 0
        if params is not None:   # (in_calib5, in_w, in_h, mode, out_calib5, out_w, out_h)
            ic, iw, ih, mode, oc, ow, oh = params
            ic = np.asarray(ic, np.float32)
            oc = np.asarray(oc if oc is not None else [0] * 5, np.float32)
            self.status = lib.mdc_fov_create_from_params(ic.ctypes.data_as(_f32p), iw, ih, mode, oc.ctypes.data_as(_f32p),
                                                         ow, oh, int(float_math), C.byref(h))
        elif configFileName is not None:
            self.status = lib.mdc_fov_create_ex(str(configFileName).encode(), int(float_math), C.byref(h))
        self._h = h if h.value else None
        self._ctx = None

    def __del__(self):
        if getattr(self, "_ctx", None) is not None:
            self._ctx.close()
        if getattr(self, "_h", None) and lib is not None:
            lib.mdc_fov_destroy(self._h)
        self._h = None

    # ---- getters (FOVUndistorter.h:49-83)
    def isValid(self) -> bool:
        return bool(self._h) and bool(lib.mdc_fov_is_valid(self._h))

    def _dims(self):
        d = [C.c_int() for _ in range(4)]
        if self._h:
            lib.mdc_fov_dims(self._h, *[C.byref(x) for x in d])
        return [x.value for x in d]

    def getInputDims(self):
        return tuple(self._dims()[:2])

    def getOutputDims(self):
        return tuple(self._dims()[2:])

    def _K(self):
        a, b = np.zeros(9, np.float32), np.zeros(9, np.float32)
        if self._h:
            lib.mdc_fov_get_K(self._h, a.ctypes.data_as(_f32p), b.ctypes.data_as(_f32p))
        return a.reshape(3, 3), b.reshape(3, 3)

    def getK_rect(self):
        return self._K()[0]

    def getK_org(self):
        return self._K()[1]

    def getOmega(self) -> float:
        return float(lib.mdc_fov_omega(self._h)) if self._h else 0.0

    def getOriginalCalibration(self):
        v = np.zeros(5, np.float32)
        if self._h:
            lib.mdc_fov_original_calibration(self._h, v.ctypes.data_as(_f32p))
        return v

    def remap_tables(self):
        """(remapX, remapY) copies — private in the reference; exposed for bit-compare / broadcast."""
        if not self.isValid():
            return None, None
        n = self.getOutputDims()[0] * self.getOutputDims()[1]
        return _np_f32(lib.mdc_fov_remap_x(self._h), n), _np_f32(lib.mdc_fov_remap_y(self._h), n)

    def distortCoordinates(self, in_x: np.ndarray, in_y: np.ndarray, n: int | None = None) -> None:
        """In place, like FOVUndistorter.cpp:280.  Prints and returns on an invalid object."""
        assert in_x.dtype == np.float32 and in_y.dtype == np.float32 and in_x.flags.c_contiguous and in_y.flags.c_contiguous
        n = in_x.size if n is None else n
        if not self._h:
            print("ERROR: invalid UndistorterFOV!")
            return
        lib.mdc_fov_distort_coordinates(self._h, in_x.ctypes.data_as(_f32p), in_y.ctypes.data_as(_f32p), n)

    def distortCoordinatesDevice(self, x, y) -> None:
        """distortCoordinates in place on float32 CUDA tensors (any number of points); bit-identical to the host version."""
        import torch
        assert x.is_cuda and y.is_cuda and x.dtype == torch.float32 and y.dtype == torch.float32
        assert x.is_contiguous() and y.is_contiguous() and x.numel() == y.numel() and x.device == y.device
        if not self._h:
            print("ERROR: invalid UndistorterFOV!")
            return
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rc = lib.mdc_fov_distort_coordinates_device(self._h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), x.numel(),
                                                    x.device.index or 0, C.c_void_p(stream))
        if rc not in (0, 4):        # 4 = MDC_ERR_INVALID_OBJECT: printed, like the reference
            check(rc, "mdc_fov_distort_coordinates_device")

    def vcPlaneMaps(self, homographies, gw: int, gh: int, p2x, p2y, facw: float = 5.0, fach: float = 5.0) -> None:
        """vignetteCalib's plane-to-image maps (main_vignetteCalib.cpp:266-284, :346-357) on the GPU: homographies float64 [n, 9]
        (or [n, 3, 3]) host array; p2x / p2y float32 CUDA tensors [n, gw*gh], overwritten (NaN = not visible)."""
        import torch
        H = np.ascontiguousarray(homographies, np.float64).reshape(-1, 9)
        n = H.shape[0]
        for t_ in (p2x, p2y):
            assert t_.is_cuda and t_.dtype == torch.float32 and t_.is_contiguous() and tuple(t_.shape) == (n, gw * gh)
        check(lib.mdc_vc_plane_maps(self._h, H.ctypes.data_as(C.POINTER(C.c_double)), n, gw, gh, float(facw), float(fach),
                                    C.c_void_p(p2x.data_ptr()), C.c_void_p(p2y.data_ptr()), p2x.device.index or 0,
                                    Context._stream(p2x)), "mdc_vc_plane_maps")

    # ---- per-frame operator (FOVUndistorter.cpp:322-370)
    def _context(self, device=0):
        if self._ctx is None:
            self._ctx = Context(self, None, device)
        return self._ctx

    def undistort(self, input, output, nPixIn: int | None = None, nPixOut: int | None = None) -> None:
        """undistort<T>(input, output, nPixIn, nPixOut); T from input dtype (uint8 / float32).
        numpy arrays = host buffers; CUDA tensors = device buffers.  Error behaviour as the
        reference: invalid object or wrong pixel counts -> message, output untouched."""
        if not self.isValid():
            return
        nPixIn = int(np.prod(input.shape)) if nPixIn is None else nPixIn
        nPixOut = int(np.prod(output.shape)) if nPixOut is None else nPixOut
        try:
            if _is_torch(input):
                ctx = self._context(input.device.index or 0)
                ctx.undistort_device(input, output, nPixIn, nPixOut)
            else:
                self._context().undistort_host(input, output, nPixIn, nPixOut)
        except MdcError as e:
            if e.code == 5:   # CUDA failure is not a reference-style soft error
                raise


class PhotometricUndistorter:
    """Photometric un-mapper (PhotometricUndistorter.h:37)."""

    def __init__(self, file: str, vignetteImage: str, w_: int, h_: int, *, arrays=None):
        h = C.c_void_p()
        self.w, self.h = w_, h_
        if arrays is not None:   # (ginv_raw256 or None, vignette pixel array or None)
            raw, vig = arrays
            rawp = np.ascontiguousarray(raw, np.float32).ctypes.data_as(_f32p) if raw is not None else None
            if vig is not None:
                vig = np.ascontiguousarray(vig)
                self.status = lib.mdc_photo_create_from_arrays(rawp, vig.ctypes.data_as(C.c_void_p), 8 if vig.dtype == np.uint8 else 16,
                                                               vig.shape[0], vig.shape[1], w_, h_, C.byref(h))
            else:
                self.status = lib.mdc_photo_create_from_arrays(rawp, None, 0, 0, 0, w_, h_, C.byref(h))
        else:
            self.status = lib.mdc_photo_create(str(file).encode(), str(vignetteImage).encode(), w_, h_, C.byref(h))
        self._h = h if h.value else None
        self._ctx = None

    def __del__(self):
        if getattr(self, "_ctx", None) is not None:
            self._ctx.close()
        if getattr(self, "_h", None) and lib is not None:
            lib.mdc_photo_destroy(self._h)
        self._h = None

    @property
    def validGamma(self) -> bool:
        return bool(self._h) and bool(lib.mdc_photo_valid_gamma(self._h))

    @property
    def validVignette(self) -> bool:
        return bool(self._h) and bool(lib.mdc_photo_valid_vignette(self._h))

    def getGInv(self):
        return _np_f32(lib.mdc_photo_ginv(self._h), 256) if self._h else None

    def getG(self):
        return _np_f32(lib.mdc_photo_g(self._h), 256) if self._h else None

    def vignette_maps(self):
        if not self.validVignette:
            return None, None
        n = self.w * self.h
        return _np_f32(lib.mdc_photo_vignette_map(self._h), n), _np_f32(lib.mdc_photo_vignette_map_inv(self._h), n)

    def _context(self, device=0):
        if self._ctx is None:
            self._ctx = Context(None, self, device)
        return self._ctx

    def unMapImage(self, image_in, image_out, n: int, undoGamma: bool, undoVignette: bool, killOverexposed: bool) -> None:
        flags = _flags(False, undoGamma, undoVignette, killOverexposed)
        if _is_torch(image_in):
            self._context(image_in.device.index or 0).unmap_device(image_in, image_out, n, flags)
        else:
            self._context().unmap_host(image_in, image_out, n, flags)


class Context:
    """Device context: calibration tables resident in HBM + tile plan (mdc_ctx)."""

    def __init__(self, fov: UndistorterFOV | None, photo: PhotometricUndistorter | None, device: int = 0, *, _adopt=None):
        h = C.c_void_p()
        self._keep = None
        if _adopt is not None:
            dims, tensors = _adopt   # (in_w, in_h, out_w, out_h), (rx, ry, ginv, vinv) CUDA tensors or None
            self._keep = tensors
            ptrs = [C.c_void_p(t.data_ptr()) if t is not None else None for t in tensors]
            check(lib.mdc_ctx_create_from_device_tables(device, *dims, *ptrs, C.byref(h)), "mdc_ctx_create_from_device_tables")
        else:
            check(lib.mdc_ctx_create(device, fov._h if fov is not None else None, photo._h if photo is not None else None,
                                     C.byref(h)), "mdc_ctx_create")
        self._h = h
        self.device = device
        self.fov, self.photo = fov, photo
        if _adopt is not None:
            self.in_dims = tuple(_adopt[0][:2])
        elif fov is not None:
            self.in_dims = tuple(fov.getInputDims())
        else:
            self.in_dims = (photo.w, photo.h) if photo is not None else (0, 0)

    @classmethod
    def from_device_tables(cls, device, in_w, in_h, out_w, out_h, rx, ry, ginv, vinv):
        """Adopt tables that were broadcast over NCCL into CUDA tensors (multi-GPU init)."""
        return cls(None, None, device, _adopt=((in_w, in_h, out_w, out_h), (rx, ry, ginv, vinv)))

    def close(self):
        if getattr(self, "_h", None) and lib is not None:   # `lib` is already gone during interpreter shutdown
            lib.mdc_ctx_destroy(self._h)
        self._h = None

    def __del__(self):
        self.close()

    LOADERS = {"auto": -1, "ldg": 0, "tma": 1, "tex": 2, "hybrid": 3}

    def configure(self, use_tma: int = -1, ctas_per_sm: int = 0):
        """use_tma: the K1 input loader, -1 auto / 0 LDG / 1 TMA / 2 texture gather (MDC_LOADER_*), or its name."""
        if isinstance(use_tma, str):
            use_tma = self.LOADERS[use_tma]
        check(lib.mdc_ctx_configure(self._h, use_tma, ctas_per_sm), "mdc_ctx_configure")

    def auto_loader(self, row_pitch: int | None = None) -> str:
        """The loader use_tma = -1 resolves to, for tightly packed rows or rows `row_pitch` bytes apart."""
        i = int(lib.mdc_ctx_auto_loader(self._h) if row_pitch is None else lib.mdc_ctx_auto_loader_pitched(self._h, row_pitch))
        return [k for k, v in self.LOADERS.items() if v == i][0]

    def loader_usable(self, loader, row_pitch: int | None = None) -> bool:
        """Whether `loader` can run on this context's frames: tightly packed rows, or rows `row_pitch` bytes apart."""
        if isinstance(loader, str):
            loader = self.LOADERS[loader]
        if row_pitch is None:
            return bool(lib.mdc_ctx_loader_usable(self._h, loader))
        return bool(lib.mdc_ctx_loader_usable_pitched(self._h, loader, row_pitch))

    @property
    def launch_count(self) -> int:
        return int(lib.mdc_ctx_launch_count(self._h))

    def level_dims(self, level: int):
        w, h = C.c_int(), C.c_int()
        check(lib.mdc_ctx_level_dims(self._h, level, C.byref(w), C.byref(h)), "mdc_ctx_level_dims")
        return w.value, h.value

    @staticmethod
    def _stream(t):
        """torch's current stream on the tensor's device as an mdc_stream.  The default stream has handle 0, which the C ABI reads as
        "the context's own stream, synchronised before returning"; torch callers mean the (legacy) default stream itself — other
        work they enqueue there, e.g. the wait torch.distributed puts behind an all-reduce, must order with ours — so it is passed
        by its explicit handle cudaStreamLegacy."""
        import torch
        h = torch.cuda.current_stream(t.device).cuda_stream
        return C.c_void_p(h if h else 0x1)

    @staticmethod
    def _drain(t):
        """Entry points without a stream argument run on the context's own stream and return when they are done; what torch has queued
        on its current stream for their inputs must be finished first."""
        import torch
        torch.cuda.current_stream(t.device).synchronize()

    # ---- device-resident operators (CUDA tensors, asynchronous on torch's current stream)
    def prepare_batch(self, frames, flags: int, out_levels, dtype=None):
        """frames: uint8 CUDA tensor [n, H*W] (or [n,H,W]); out_levels: list of CUDA tensors of `dtype` (torch.float32 (default),
        torch.float16 or torch.uint8: the fp32 levels converted as MDC_OUT_F16 / MDC_OUT_U8 describe, inside the same kernels)."""
        self._prepare(frames, 0, flags, out_levels, dtype)

    def prepare_batch_pitched(self, frames, pitch: int, flags: int, out_levels, dtype=None):
        """frames: uint8 CUDA tensor [n, H, pitch] whose rows hold in_w pixels followed by padding (rectifying mode only).
        out_levels and dtype as for prepare_batch."""
        if pitch == 0:
            raise ValueError("prepare_batch_pitched: row pitch 0 (use prepare_batch for tightly packed rows)")
        self._prepare(frames, pitch, flags, out_levels, dtype)

    def _prepare(self, frames, pitch, flags, out_levels, dtype):
        out_type = _out_type(dtype)
        _check_out_dtype(out_levels, dtype)
        n = frames.shape[0]
        arr = (C.c_void_p * len(out_levels))(*[t.data_ptr() for t in out_levels])
        check(lib.mdc_prepare_batch_ex(self._h, C.c_void_p(frames.data_ptr()), pitch, n, flags, out_type, arr, len(out_levels),
                                       self._stream(frames)), "mdc_prepare_batch")

    def unmap_device(self, image_in, image_out, n, flags, n_frames=1):
        check(lib.mdc_unmap_u8(self._h, C.c_void_p(image_in.data_ptr()), C.c_void_p(image_out.data_ptr()), n, n_frames, flags,
                               self._stream(image_in)), "mdc_unmap_u8")

    def undistort_device(self, inp, out, n_in, n_out, n_frames=1):
        import torch
        fn = lib.mdc_undistort_u8 if inp.dtype == torch.uint8 else lib.mdc_undistort_f32
        check(fn(self._h, C.c_void_p(inp.data_ptr()), C.c_void_p(out.data_ptr()), n_in, n_out, n_frames, self._stream(inp)),
              "mdc_undistort")

    def pyr_down(self, src, sw, sh, dst, n_frames=1):
        check(lib.mdc_pyr_down(self._h, C.c_void_p(src.data_ptr()), sw, sh, C.c_void_p(dst.data_ptr()), n_frames, self._stream(src)),
              "mdc_pyr_down")

    def estep(self, data, t, G, E):
        """data uint8 [n, npix], t float64 [n], G float64 [256] -> E float64 [npix] (all CUDA tensors)."""
        check(lib.mdc_estep(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()),
                            C.c_void_p(G.data_ptr()), C.c_void_p(E.data_ptr()), self._stream(data)), "mdc_estep")

    # ---- responseCalib building blocks (CUDA tensors; main_responseCalib.cpp)
    def rc_leak_padding(self, data, w, h, iterations):
        check(lib.mdc_rc_leak_padding(self._h, C.c_void_p(data.data_ptr()), data.shape[0], w, h, iterations, self._stream(data)), "mdc_rc_leak_padding")

    def rc_einit(self, data, E):
        check(lib.mdc_rc_einit(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(E.data_ptr()), self._stream(data)), "mdc_rc_einit")

    def rc_gstep(self, data, t, E, G):
        check(lib.mdc_rc_gstep(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()),
                               C.c_void_p(E.data_ptr()), C.c_void_p(G.data_ptr()), self._stream(data)), "mdc_rc_gstep")

    def rc_rescale(self, E, G) -> float:
        self._drain(E)
        f = C.c_double()
        check(lib.mdc_rc_rescale(self._h, E.shape[0], C.c_void_p(E.data_ptr()), C.c_void_p(G.data_ptr()), C.byref(f)), "mdc_rc_rescale")
        return f.value

    def rc_rmse(self, data, t, G, E):
        self._drain(data)
        out = (C.c_double * 2)()
        check(lib.mdc_rc_rmse(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()),
                              C.c_void_p(G.data_ptr()), C.c_void_p(E.data_ptr()), out), "mdc_rc_rmse")
        return out[0], out[1]

    # the two reductions as per-rank partials (pixel-sharded runs; accumulators are CUDA tensors: gsum f64[256], gnum i64[256], acc f64[2])
    def rc_gstep_accumulate(self, data, t, E, gsum, gnum, reuse_counts=False):
        check(lib.mdc_rc_gstep_accumulate(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()),
                                          C.c_void_p(E.data_ptr()), C.c_void_p(gsum.data_ptr()), C.c_void_p(gnum.data_ptr()),
                                          int(bool(reuse_counts)), self._stream(data)), "mdc_rc_gstep_accumulate")

    def rc_gstep_finish(self, gsum, gnum, G):
        check(lib.mdc_rc_gstep_finish(self._h, C.c_void_p(gsum.data_ptr()), C.c_void_p(gnum.data_ptr()), C.c_void_p(G.data_ptr()),
                                      self._stream(G)), "mdc_rc_gstep_finish")

    # the G-step with sums that are exact across ranks: scale4 i64[4] (all-reduce MAX), limbs i64[768] + special f64[256] (all-reduce SUM)
    def rc_gstep_scale(self, E, t, scale4):
        check(lib.mdc_rc_gstep_scale(self._h, C.c_void_p(E.data_ptr()), E.shape[0], C.c_void_p(t.data_ptr()), t.shape[0],
                                     C.c_void_p(scale4.data_ptr()), self._stream(E)), "mdc_rc_gstep_scale")

    def rc_gstep_accumulate_exact(self, data, t, E, scale4, limbs, special, gnum, reuse_counts=False):
        check(lib.mdc_rc_gstep_accumulate_exact(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()),
                                                C.c_void_p(E.data_ptr()), C.c_void_p(scale4.data_ptr()), C.c_void_p(limbs.data_ptr()),
                                                C.c_void_p(special.data_ptr()), C.c_void_p(gnum.data_ptr()), int(bool(reuse_counts)),
                                                self._stream(data)), "mdc_rc_gstep_accumulate_exact")

    def rc_gstep_finish_exact(self, scale4, limbs, special, gnum, G):
        check(lib.mdc_rc_gstep_finish_exact(self._h, C.c_void_p(scale4.data_ptr()), C.c_void_p(limbs.data_ptr()), C.c_void_p(special.data_ptr()),
                                            C.c_void_p(gnum.data_ptr()), C.c_void_p(G.data_ptr()), self._stream(G)), "mdc_rc_gstep_finish_exact")

    def rc_rmse_accumulate(self, data, t, G, E, acc):
        check(lib.mdc_rc_rmse_accumulate(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()),
                                         C.c_void_p(G.data_ptr()), C.c_void_p(E.data_ptr()), C.c_void_p(acc.data_ptr()), self._stream(data)),
              "mdc_rc_rmse_accumulate")

    def response_calib(self, data, t, nits, E, G, on_step=None):
        """The optimisation loop of responseCalib's main(); returns the per-iteration log [nits, 4].
        on_step(iteration, which, E, G), if given, is called where the reference plots: after E-init (0, "E"), and in iteration it
        after the G-step (it + 1, "G") and after the E-step, before the rescale (it + 1, "E").  E and G hold that step's values; the
        callback may read them, copy them or run the plots on them (rc_plot_e, rc_plot_g) but must not change them.  Work it enqueues
        on torch's current stream is finished before the loop goes on (the loop writes E and G in place on the context's own stream),
        so a snapshot such as E.clone() holds that step's values."""
        self._drain(data)
        log = np.zeros((max(nits, 1), 4), np.float64)
        failed = []

        def step(iteration, which, _e, _g, _user):
            if failed:
                return
            try:
                on_step(iteration, "G" if which == _lib.RC_STEP_G else "E", E, G)
            except BaseException as exc:              # raised again below: an exception cannot cross the C frames
                failed.append(exc)
            finally:
                self._drain(E)                        # the next pass overwrites E / G without waiting for torch's stream

        hook = _lib.RC_STEP_FN(step) if on_step is not None else None
        check(lib.mdc_response_calib_ex(self._h, C.c_void_p(data.data_ptr()), data.shape[0], data.shape[1], C.c_void_p(t.data_ptr()), nits,
                                        C.c_void_p(E.data_ptr()), C.c_void_p(G.data_ptr()), log.ctypes.data_as(C.POINTER(C.c_double)),
                                        C.cast(hook, C.c_void_p) if hook else None, None), "mdc_response_calib_ex")
        if failed:
            raise failed[0]
        return log[:nits]

    # ---- responseCalib's result images (main_responseCalib.cpp:72-146; CUDA tensors, on torch's current stream)
    def rc_plot_e_range(self, E, range4=None):
        """{min ln(E+20), max ln(E+20), min E, max E} of a float64 CUDA tensor (any shape) into a float64 CUDA tensor [4] (new when
        range4 is None).  The ranges of slices join into the range of the whole image by strict min / max taken in slice order
        (rc_plot_join_ranges)."""
        import torch
        assert E.is_cuda and E.dtype == torch.float64 and E.is_contiguous()
        range4 = torch.empty(4, dtype=torch.float64, device=E.device) if range4 is None else range4
        assert range4.is_cuda and range4.dtype == torch.float64 and range4.numel() == 4
        check(lib.mdc_rc_plot_e_range(self._h, C.c_void_p(E.data_ptr()), E.numel(), C.c_void_p(range4.data_ptr()), self._stream(E)),
              "mdc_rc_plot_e_range")
        return range4

    def rc_plot_e_map(self, E, range4, bgr=None, e16=None):
        """plotE's two images of E under the range range4 (a CUDA tensor): bgr uint8 [npix, 3] (BGR order) and e16 uint16 [npix]."""
        import torch
        assert E.is_cuda and E.dtype == torch.float64 and E.is_contiguous()
        assert range4.is_cuda and range4.dtype == torch.float64 and range4.numel() == 4
        n = E.numel()
        bgr = torch.empty((n, 3), dtype=torch.uint8, device=E.device) if bgr is None else bgr
        e16 = torch.empty(n, dtype=torch.uint16, device=E.device) if e16 is None else e16
        assert bgr.is_cuda and bgr.dtype == torch.uint8 and bgr.is_contiguous() and bgr.numel() == 3 * n
        assert e16.is_cuda and e16.dtype == torch.uint16 and e16.is_contiguous() and e16.numel() == n
        check(lib.mdc_rc_plot_e_map(self._h, C.c_void_p(E.data_ptr()), n, C.c_void_p(range4.data_ptr()), C.c_void_p(bgr.data_ptr()),
                                    C.c_void_p(e16.data_ptr()), self._stream(E)), "mdc_rc_plot_e_map")
        return bgr, e16

    def rc_plot_e(self, E, w, h):
        """plotE (E-k.png, E-k16.png) of a w x h irradiance: (bgr uint8 CUDA [h, w, 3] in BGR order, e16 uint16 CUDA [h, w],
        (min ln(E+20), max ln(E+20), min E, max E))."""
        assert E.numel() == w * h
        range4 = self.rc_plot_e_range(E)
        bgr, e16 = self.rc_plot_e_map(E, range4)
        return bgr.view(h, w, 3), e16.view(h, w), tuple(range4.tolist())

    def rc_plot_g(self, G):
        """plotG (G-k.png) of a float64 CUDA tensor [256]: (uint8 CUDA [256, 256], (min G, max G))."""
        import torch
        assert G.is_cuda and G.dtype == torch.float64 and G.is_contiguous() and G.numel() == 256
        out = torch.empty((256, 256), dtype=torch.uint8, device=G.device)
        mm = (C.c_double * 2)()
        check(lib.mdc_rc_plot_g(self._h, C.c_void_p(G.data_ptr()), C.c_void_p(out.data_ptr()), mm, self._stream(G)), "mdc_rc_plot_g")
        return out, (mm[0], mm[1])

    # ---- vignetteCalib optimiser (CUDA tensors; main_vignetteCalib.cpp:395-585)
    @staticmethod
    def _vc_dims(images, p2x, p2y, gw, gh, wI, hI):
        import torch
        n = p2x.shape[0]
        for t_, cols in ((images, wI * hI), (p2x, gw * gh), (p2y, gw * gh)):
            assert t_.is_cuda and t_.dtype == torch.float32 and t_.is_contiguous() and tuple(t_.shape) == (n, cols)
        return n

    def vc_prepare_images(self, raw, wI, hI, exposures, mean_exposure, max_abs_grad=255, out=None):
        """Exposure normalisation + gradient invalidation (main_vignetteCalib.cpp:286-301): raw float32 CUDA tensor [n, wI*hI],
        exposures [n] (host); out defaults to a new tensor and may be raw itself.  Returns out."""
        import torch
        n = raw.shape[0]
        out = torch.empty_like(raw) if out is None else out
        for t_ in (raw, out):
            assert t_.is_cuda and t_.dtype == torch.float32 and t_.is_contiguous() and tuple(t_.shape) == (n, wI * hI)
        t = np.ascontiguousarray(np.asarray(exposures, np.float32).reshape(-1))
        assert t.size == n
        check(lib.mdc_vc_prepare_images(self._h, C.c_void_p(raw.data_ptr()), n, wI, hI, t.ctypes.data_as(_f32p), float(mean_exposure),
                                        int(max_abs_grad), C.c_void_p(out.data_ptr()), self._stream(raw)), "mdc_vc_prepare_images")
        return out

    def vc_plane_step(self, images, p2x, p2y, gw, gh, wI, hI, vignette, plane_color, oth2, integer_abs=True):
        """plane_color is updated in place; returns (E, R)."""
        self._drain(images)
        import torch
        n = self._vc_dims(images, p2x, p2y, gw, gh, wI, hI)
        st = (C.c_double * 2)()
        check(lib.mdc_vc_plane_step(self._h, C.c_void_p(images.data_ptr()), C.c_void_p(p2x.data_ptr()), C.c_void_p(p2y.data_ptr()), n, gw, gh, wI, hI,
                                    C.c_void_p(vignette.data_ptr()), C.c_void_p(plane_color.data_ptr()), float(oth2), int(integer_abs), st), "mdc_vc_plane_step")
        return st[0], st[1]

    def vc_vignette_step(self, images, p2x, p2y, gw, gh, wI, hI, plane_color, vignette, oth2, integer_abs=True):
        """vignette is updated in place (normalised to maximum 1); returns (E, R)."""
        self._drain(images)
        import torch
        n = self._vc_dims(images, p2x, p2y, gw, gh, wI, hI)
        st = (C.c_double * 2)()
        check(lib.mdc_vc_vignette_step(self._h, C.c_void_p(images.data_ptr()), C.c_void_p(p2x.data_ptr()), C.c_void_p(p2y.data_ptr()), n, gw, gh, wI, hI,
                                       C.c_void_p(plane_color.data_ptr()), C.c_void_p(vignette.data_ptr()), float(oth2), int(integer_abs), st), "mdc_vc_vignette_step")
        return st[0], st[1]

    def vc_smooth(self, vignette, wI, hI, iterations=4):
        self._drain(vignette)
        import torch
        out = torch.empty_like(vignette)
        check(lib.mdc_vc_smooth(self._h, C.c_void_p(vignette.data_ptr()), wI, hI, iterations, C.c_void_p(out.data_ptr())), "mdc_vc_smooth")
        return out

    def vignette_calib(self, images, p2x, p2y, gw, gh, wI, hI, max_iterations, outlier_th, plane_color, vignette, integer_abs=True):
        """The reference's optimisation loop; plane_color / vignette updated in place.  Returns (smoothed vignette, log [its, 4])."""
        self._drain(images)
        import torch
        n = self._vc_dims(images, p2x, p2y, gw, gh, wI, hI)
        smoothed = torch.empty_like(vignette)
        log = np.zeros((max(max_iterations, 1), 4), np.float64)
        check(lib.mdc_vignette_calib(self._h, C.c_void_p(images.data_ptr()), C.c_void_p(p2x.data_ptr()), C.c_void_p(p2y.data_ptr()), n, gw, gh, wI, hI,
                                     max_iterations, outlier_th, int(integer_abs), C.c_void_p(plane_color.data_ptr()), C.c_void_p(vignette.data_ptr()),
                                     C.c_void_p(smoothed.data_ptr()), log.ctypes.data_as(C.POINTER(C.c_double))), "mdc_vignette_calib")
        return smoothed, log[:max_iterations]

    # ---- host-buffer operators (numpy)
    def marker_threshold(self, rect, grey=None, mask=None):
        """vignetteCalib's 8-bit conversion and aruco's adaptive threshold on the GPU (mdc_marker_threshold): rect float32 CUDA tensor
        [n, h, w] of rectified frames; grey, mask uint8 [n, h, w] (new tensors when None).  Returns (grey, mask)."""
        import torch
        n, h, w = rect.shape
        grey = torch.empty(rect.shape, dtype=torch.uint8, device=rect.device) if grey is None else grey
        mask = torch.empty(rect.shape, dtype=torch.uint8, device=rect.device) if mask is None else mask
        assert rect.is_cuda and rect.dtype == torch.float32 and rect.is_contiguous()
        for t_ in (grey, mask):
            assert t_.is_cuda and t_.dtype == torch.uint8 and t_.is_contiguous() and tuple(t_.shape) == (n, h, w)
        check(lib.mdc_marker_threshold(self._h, C.c_void_p(rect.data_ptr()), n, w, h, C.c_void_p(grey.data_ptr()),
                                       C.c_void_p(mask.data_ptr()), self._stream(rect)), "mdc_marker_threshold")
        return grey, mask

    def unmap_host(self, image_in: np.ndarray, image_out: np.ndarray, n, flags):
        assert image_in.dtype == np.uint8 and image_out.dtype == np.float32
        check(lib.mdc_unmap_u8_host(self._h, image_in.ctypes.data_as(C.c_void_p), image_out.ctypes.data_as(C.c_void_p), n, flags),
              "mdc_unmap_u8_host")

    def undistort_host(self, inp: np.ndarray, out: np.ndarray, n_in, n_out):
        assert out.dtype == np.float32 and inp.dtype in (np.uint8, np.float32)
        fn = lib.mdc_undistort_u8_host if inp.dtype == np.uint8 else lib.mdc_undistort_f32_host
        check(fn(self._h, inp.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), n_in, n_out), "mdc_undistort_host")

    def prepare_batch_host(self, frames, flags: int, out_levels, dtype=None):
        """frames / out_levels: numpy arrays or raw integer addresses of (pinned) host memory; the levels hold `dtype` elements
        (np.float32 (default), np.float16 or np.uint8, or the torch dtypes of those)."""
        def addr(x):
            return x if isinstance(x, int) else x.ctypes.data
        out_type = _out_type(dtype)
        _check_out_dtype(out_levels, dtype)
        n = frames.shape[0]
        arr = (C.c_void_p * len(out_levels))(*[addr(t) for t in out_levels])
        check(lib.mdc_prepare_batch_host_ex(self._h, C.c_void_p(addr(frames)), n, flags, out_type, arr, len(out_levels)),
              "mdc_prepare_batch_host")


class ExposureImage:
    """ExposureImage.h:33 — float image + metadata (numpy-owned)."""

    def __init__(self, w_, h_, timestamp_, exposure_, id_):
        self.w, self.h, self.timestamp, self.exposure_time, self.id = w_, h_, timestamp_, exposure_, id_
        self.image = np.empty(w_ * h_, np.float32)


class Sequence:
    """The file side of DatasetReader (BenchmarkDatasetReader.h:83-147, :159-186, :247-345): images/ folder or images.zip, times.txt,
    raw 8-bit frames (lossless formats: PNG, PGM), and the decode-ahead feed of the GPU path (SURVEY.md §8f N1)."""

    def __init__(self, folder: str):
        h = C.c_void_p()
        self.status = lib.mdc_seq_open(folder.encode(), C.byref(h))
        self._h = h if self.status == 0 else None

    def close(self):
        if getattr(self, "_h", None) is not None and lib is not None:
            lib.mdc_seq_close(self._h)
        self._h = None

    __del__ = close

    def getNumImages(self) -> int:
        return lib.mdc_seq_num_images(self._h) if self._h else 0

    def isZipped(self) -> bool:
        return bool(lib.mdc_seq_is_zipped(self._h)) if self._h else False

    def name(self, id_: int):
        v = lib.mdc_seq_name(self._h, id_) if self._h else None
        return v.decode() if v else None

    def getTimestamp(self, id_: int) -> float:
        return lib.mdc_seq_timestamp(self._h, id_) if self._h else 0.0

    def getExposure(self, id_: int) -> float:
        return lib.mdc_seq_exposure(self._h, id_) if self._h else 0.0

    def getImageRaw_internal(self, id_: int):
        """Decoded 8-bit grey frame [h, w], or None if it cannot be decoded (cv::imread would return an empty Mat)."""
        if not self._h:
            return None
        w, h = C.c_int(), C.c_int()
        guess = getattr(self, "_last_shape", None)
        if guess is not None:                       # frames of a sequence share one size: try a buffer of that size first
            out = np.empty(guess, np.uint8)
            rc = lib.mdc_seq_read_gray8(self._h, id_, out.ctypes.data_as(C.c_void_p), out.size, C.byref(w), C.byref(h))
            if rc == 0 and (h.value, w.value) == guess:
                return out
        if lib.mdc_seq_read_gray8(self._h, id_, None, 0, C.byref(w), C.byref(h)) != 0:
            return None
        out = np.empty((h.value, w.value), np.uint8)
        check(lib.mdc_seq_read_gray8(self._h, id_, out.ctypes.data_as(C.c_void_p), out.size, C.byref(w), C.byref(h)), "mdc_seq_read_gray8")
        self._last_shape = (h.value, w.value)
        return out

    def prepare(self, ctx: "Context", level_shapes, first: int, count: int, rectify, removeGamma, removeVignette, nanOverexposed,
                threads: int = 0, dtype=None):
        """getImage for frames [first, first+count) -> list of arrays [count, w_l*h_l] (one per pyramid level) of `dtype`
        (np.float32 (default), np.float16 or np.uint8)."""
        out_type = _out_type(dtype)
        outs = [np.empty((count, w * h), _dtype_name(dtype)) for (w, h) in level_shapes]
        ptrs = (C.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
        check(lib.mdc_seq_prepare_ex(ctx._h, self._h, first, count, _flags(rectify, removeGamma, removeVignette, nanOverexposed), out_type, ptrs,
                                     len(outs), threads), "mdc_seq_prepare")
        return outs

    def prepare_device(self, ctx: "Context", first: int, count: int, rectify, removeGamma, removeVignette, nanOverexposed, levels: int = 1,
                       threads: int = 0, out=None, dtype=None):
        """getImage for frames [first, first+count) with the JPEG frames decoded on the GPU (mdc_seq_prepare_device) -> list of CUDA
        tensors [count, w_l*h_l] of `dtype` (torch.float32 (default), torch.float16 or torch.uint8) on the context's device, one per
        pyramid level.  Runs on torch's current stream."""
        import torch
        out_type = _out_type(dtype)
        if out is None:
            w, h = ctx.level_dims(0) if rectify else ctx.in_dims
            tdt = getattr(torch, _dtype_name(dtype))
            out = [torch.empty((count, (w >> l) * (h >> l)), dtype=tdt, device=f"cuda:{ctx.device}") for l in range(levels)]
        _check_out_dtype(out, dtype)
        ptrs = (C.c_void_p * len(out))(*[t.data_ptr() for t in out])
        stream = Context._stream(out[0]) if out else None
        check(lib.mdc_seq_prepare_device_ex(ctx._h, self._h, first, count, _flags(rectify, removeGamma, removeVignette, nanOverexposed), out_type,
                                            ptrs, len(out), threads, stream), "mdc_seq_prepare_device")
        return out

    def read_gray8_device(self, ctx: "Context", ids, w: int, h: int, row_pitch: int | None = None, threads: int = 0, out=None):
        """getImageRaw_internal(id) for every id (any order, repeats allowed), decoded into device memory (mdc_seq_read_gray8_device) ->
        (uint8 CUDA tensor [n, h, row_pitch] on the context's device, status int32 [n], sizes int32 [n, 2]).  Per frame, as
        mdc_seq_read_gray8: status 0 = read at w x h; 3 = MDC_ERR_FORMAT, it cannot be read; 1 = MDC_ERR_INVALID_ARG, it reads at
        another size.  sizes holds (w, h) as the host reader reports them, (0, 0) if it cannot read the frame.  Rows of a frame that
        is not read, and the padding of every row, keep what `out` held.  row_pitch defaults to w rounded up to 16 bytes.  Runs on
        torch's current stream; bad arguments and runtime failures raise MdcError."""
        import torch
        ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
        n = ids.size
        pitch = row_pitch if row_pitch is not None else (w + 15) // 16 * 16
        if out is None:
            out = torch.zeros((n, h, pitch), dtype=torch.uint8, device=f"cuda:{ctx.device}")
        elif out.dtype != torch.uint8 or not out.is_cuda or not out.is_contiguous() or tuple(out.shape) != (n, h, pitch):
            raise ValueError(f"out must be a contiguous uint8 CUDA tensor of shape {(n, h, pitch)}")
        status = np.zeros(n, np.int32)
        sizes = np.zeros((n, 2), np.int32)
        rc = lib.mdc_seq_read_gray8_device(ctx._h, self._h, ids.ctypes.data, n, w, h, C.c_void_p(out.data_ptr()), pitch, status.ctypes.data,
                                           sizes.ctypes.data, threads, Context._stream(out))
        if rc not in (0, 3):
            check(rc, "mdc_seq_read_gray8_device")
        return out, status, sizes


class FramePreparer:
    """The getImage composition of DatasetReader (BenchmarkDatasetReader.h:188-243) over frames that are already decoded
    (use Sequence for the folder / zip / times.txt side)."""

    def __init__(self, undistorter: UndistorterFOV, photoUndistorter: PhotometricUndistorter, device: int = 0):
        self.undistorter, self.photoUndistorter = undistorter, photoUndistorter
        self.widthOrg, self.heightOrg = undistorter.getInputDims()
        self.width, self.height = undistorter.getOutputDims()
        self.ctx = Context(undistorter, photoUndistorter, device)

    def getUndistorter(self):
        return self.undistorter

    def getPhotoUndistorter(self):
        return self.photoUndistorter

    def getImage(self, imageRaw: np.ndarray, id_: int, rectify: bool, removeGamma: bool, removeVignette: bool,
                 nanOverexposed: bool, timestamp: float = 0.0, exposure: float = 0.0):
        """One decoded 8-bit frame -> ExposureImage, or None on a dimension/type mismatch (:194-205)."""
        if imageRaw.ndim != 2 or imageRaw.shape != (self.heightOrg, self.widthOrg):
            shp = imageRaw.shape if imageRaw.ndim == 2 else (0, 0)
            print("ERROR: expected cv-mat to have dimensions %d x %d; found %d x %d (image %d)!" %
                  (self.widthOrg, self.heightOrg, shp[1], shp[0], id_))
            return None
        if imageRaw.dtype != np.uint8:
            print("ERROR: expected cv-mat to have type 8U!")
            return None
        w, h = (self.width, self.height) if rectify else (self.widthOrg, self.heightOrg)
        ret = ExposureImage(w, h, timestamp, exposure, id_)
        raw = np.ascontiguousarray(imageRaw).reshape(1, -1)
        self.ctx.prepare_batch_host(raw, _flags(rectify, removeGamma, removeVignette, nanOverexposed), [ret.image])
        return ret

    def level_shapes(self, rectify: bool, levels: int):
        w, h = (self.width, self.height) if rectify else (self.widthOrg, self.heightOrg)
        return [(w >> l, h >> l) for l in range(levels)]

    def prepare_device(self, frames, rectify, removeGamma, removeVignette, nanOverexposed, levels: int = 1, out=None, dtype=None):
        """Batched, device-resident getImage (+ pyramid): frames uint8 CUDA tensor [n, H*W]; levels of `dtype` (torch.float32 (default),
        torch.float16 or torch.uint8)."""
        import torch
        _out_type(dtype)
        n = frames.shape[0]
        if out is None:
            tdt = getattr(torch, _dtype_name(dtype))
            out = [torch.empty((n, w * h), dtype=tdt, device=frames.device) for (w, h) in self.level_shapes(rectify, levels)]
        self.ctx.prepare_batch(frames, _flags(rectify, removeGamma, removeVignette, nanOverexposed), out, dtype=dtype)
        return out


def jpeg_decode_device(blobs, w: int, h: int, ctx: "Context | None" = None, device: int = 0, row_pitch: int | None = None, out=None):
    """Baseline JPEG files (bytes) -> uint8 CUDA tensor [n, h, row_pitch] of grey planes decoded on the GPU (mdc_jpeg_decode_device), the
    same bytes as the host decoder, and the per-frame status (0 = decoded, 3 = MDC_ERR_FORMAT: that frame's rows are left as they were).
    row_pitch defaults to w rounded up to 16 bytes.  Errors other than undecodable frames raise MdcError."""
    import torch
    if ctx is None:
        ctx = Context(None, None, device)
    n = len(blobs)
    pitch = row_pitch if row_pitch is not None else (w + 15) // 16 * 16
    if out is None:
        out = torch.zeros((n, h, pitch), dtype=torch.uint8, device=f"cuda:{ctx.device}")
    keep = [bytes(b) for b in blobs]
    files = (C.c_void_p * max(n, 1))(*[C.cast(C.c_char_p(b), C.c_void_p).value for b in keep])
    sizes = (C.c_size_t * max(n, 1))(*[len(b) for b in keep])
    status = (C.c_int * max(n, 1))()
    rc = lib.mdc_jpeg_decode_device(ctx._h, files, sizes, n, w, h, C.c_void_p(out.data_ptr()), pitch, status, Context._stream(out))
    if rc not in (0, 3):
        check(rc, "mdc_jpeg_decode_device")
    return out, np.array(status[:n], dtype=np.int32)


def jpeg_encode_bound(w: int, h: int) -> int:
    """Bytes the JPEG file of a w x h frame can take at any quality (mdc_jpeg_encode_bound)."""
    return int(lib.mdc_jpeg_encode_bound(w, h))


def jpeg_encode_device(frames, quality: int = 95, ctx: "Context | None" = None, device: int = 0, row_pitch: int | None = None) -> list:
    """cv2.imencode('.jpg', frame, [cv2.IMWRITE_JPEG_QUALITY, quality]) of every frame, encoded on the GPU (mdc_jpeg_encode_device):
    frames is a uint8 CUDA tensor [n, h, w] whose rows may be padded, e.g. a [:, :, :w] slice of a [n, h, pitch] buffer; the padding is
    never read.  row_pitch defaults to the tensor's row stride.  Runs on torch's current stream; returns the n files as bytes."""
    import torch
    if frames.dtype != torch.uint8 or not frames.is_cuda or frames.dim() != 3 or (frames.shape[0] and frames.shape[2] and frames.stride(2) != 1):
        raise ValueError("jpeg_encode_device: frames must be a uint8 CUDA tensor [n, h, w] with unit stride along w")
    n, h, w = frames.shape
    pitch = row_pitch if row_pitch is not None else frames.stride(1)
    if n > 1 and frames.stride(0) != h * pitch:
        raise ValueError("jpeg_encode_device: frames must be h * row_pitch bytes apart")
    if ctx is None:
        ctx = Context(None, None, frames.device.index if frames.device.index is not None else device)
    stride = jpeg_encode_bound(w, h)
    out = torch.empty((n, max(stride, 1)), dtype=torch.uint8, device=frames.device)
    sizes = (C.c_size_t * max(n, 1))()
    check(lib.mdc_jpeg_encode_device(ctx._h, C.c_void_p(frames.data_ptr()), pitch, n, w, h, quality, C.c_void_p(out.data_ptr()), stride,
                                     sizes, Context._stream(out)), "mdc_jpeg_encode_device")
    if n == 0:
        return []
    packed = torch.cat([out[k, :sizes[k]] for k in range(n)]).cpu().numpy().tobytes()      # only the files' bytes cross to the host
    ends = np.cumsum([sizes[k] for k in range(n)])
    return [packed[e - sizes[k]:e] for k, e in enumerate(ends)]


def atanf_host(x: np.ndarray) -> np.ndarray:
    """The restated glibc atanf (csrc/mdc_atanf.h) evaluated on the host."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.empty_like(x)
    lib.mdc_atanf_host(x.ctypes.data_as(_f32p), out.ctypes.data_as(_f32p), x.size)
    return out


def atanf_device(x):
    """The same function evaluated by the GPU (float32 CUDA tensor in, new tensor out)."""
    import torch
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty_like(x)
    check(lib.mdc_atanf_device(C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), x.numel(), x.device.index or 0,
                               C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)), "mdc_atanf_device")
    return out


def rc_plot_join_ranges(ranges):
    """The range of a whole image from the ranges of its pixel slices (rc_plot_e_range of each), given in slice order: strict
    min / max from the starting values 1e10 / -1e10, so an earlier slice keeps a tie, as the reference's scan keeps the first of
    +0 and -0.  Returns [min ln(E+20), max ln(E+20), min E, max E] as Python floats."""
    out = [1e10, -1e10, 1e10, -1e10]
    for r in ranges:
        r = [float(v) for v in (r.tolist() if hasattr(r, "tolist") else r)]
        for k in range(4):
            if (r[k] > out[k]) if k & 1 else (r[k] < out[k]):
                out[k] = r[k]
    return out


def libm_host(x: np.ndarray, op: str) -> np.ndarray:
    """glibc's double exp or log as the plots evaluate them (csrc/mdc_libm.h), on the host; op is "exp" or "log"."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty_like(x)
    lib.mdc_libm_host(_lib.LIBM_EXP if op == "exp" else _lib.LIBM_LOG, x.ctypes.data, out.ctypes.data, x.size)
    return out


def libm_device(x, op: str):
    """The same functions evaluated by the GPU (float64 CUDA tensor in, new tensor out)."""
    import torch
    assert x.is_cuda and x.dtype == torch.float64 and x.is_contiguous() and op in ("exp", "log")
    out = torch.empty_like(x)
    check(lib.mdc_libm_device(_lib.LIBM_EXP if op == "exp" else _lib.LIBM_LOG, C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()),
                              x.numel(), x.device.index or 0, C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)), "mdc_libm_device")
    return out


def png_write(path: str, img: np.ndarray) -> None:
    """Write a uint8 or uint16 image [h, w] (grey) or [h, w, 3] (BGR, as cv2.imwrite takes it) as a PNG file; rows may be strided."""
    assert img.dtype in (np.uint8, np.uint16) and img.ndim in (2, 3) and (img.ndim == 2 or img.shape[2] == 3)
    if img.strides[0] < 0 or img.strides[-1] != img.itemsize or (img.ndim == 3 and img.strides[1] != 3 * img.itemsize):
        img = np.ascontiguousarray(img)
    check(lib.mdc_png_write(path.encode(), img.ctypes.data, img.shape[1], img.shape[0], img.strides[0], 8 * img.itemsize,
                            1 if img.ndim == 2 else 3), "mdc_png_write")


class _Marker(C.Structure):
    _fields_ = [("id", C.c_int), ("corners", C.c_float * 8)]


def _u8_image(a, name):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    assert a.ndim == 2, f"{name} must be [h, w]"
    return a


def marker_detect(grey: np.ndarray, mask: np.ndarray, capacity: int = 64):
    """aruco's MarkerDetector::detect from the 8-bit frame and its threshold mask (mdc_marker_detect), both uint8 [h, w]:
    a list of (id, corners float32 [4, 2]) sorted by id."""
    grey, mask = _u8_image(grey, "grey"), _u8_image(mask, "mask")
    assert grey.shape == mask.shape
    h, w = grey.shape
    out = (_Marker * max(capacity, 1))()
    count = C.c_int()
    check(lib.mdc_marker_detect(grey.ctypes.data, mask.ctypes.data, w, h, out, capacity, C.byref(count)), "mdc_marker_detect")
    return [(out[i].id, np.array(out[i].corners, np.float32).reshape(4, 2)) for i in range(count.value)]


def marker_homography(corners) -> np.ndarray:
    """vignetteCalib's homography from the unit square to the four marker corners (mdc_marker_homography): float64 [3, 3]."""
    c = np.ascontiguousarray(np.asarray(corners, np.float32).reshape(8))
    H = (C.c_double * 9)()
    check(lib.mdc_marker_homography(c.ctypes.data_as(_f32p), H), "mdc_marker_homography")
    return np.array(H[:], np.float64).reshape(3, 3)


def marker_contours(mask: np.ndarray):
    """The contours mdc_marker_detect traces (mdc_marker_contours), in findContours's order: a list of int32 [n, 2] arrays (x, y)."""
    mask = _u8_image(mask, "mask")
    h, w = mask.shape
    nc, npt = C.c_int(), C.c_size_t()
    lib.mdc_marker_contours(mask.ctypes.data, w, h, None, 0, None, 0, C.byref(nc), C.byref(npt))
    xy = np.empty((max(npt.value, 1), 2), np.int32)
    lengths = np.empty(max(nc.value, 1), np.int32)
    check(lib.mdc_marker_contours(mask.ctypes.data, w, h, xy.ctypes.data, npt.value, lengths.ctypes.data, nc.value, C.byref(nc),
                                  C.byref(npt)), "mdc_marker_contours")
    ends = np.cumsum(lengths[:nc.value])
    return [xy[e - n:e].copy() for e, n in zip(ends, lengths[:nc.value])]


def marker_approx_poly(points, eps: float) -> np.ndarray:
    """approxPolyDP(points, eps, closed=True) as mdc_marker_detect computes it: int32 [m, 2]."""
    p = np.ascontiguousarray(np.asarray(points, np.int32).reshape(-1, 2))
    out = np.empty((max(len(p), 1), 2), np.int32)
    n = C.c_int()
    check(lib.mdc_marker_approx_poly(p.ctypes.data, len(p), float(eps), out.ctypes.data, C.byref(n)), "mdc_marker_approx_poly")
    return out[:n.value].copy()


def marker_candidates(mask: np.ndarray, capacity: int = 4096) -> np.ndarray:
    """The quads detectRectangles keeps (mdc_marker_candidates): float32 [count, 4, 2]."""
    mask = _u8_image(mask, "mask")
    h, w = mask.shape
    out = np.empty((max(capacity, 1), 4, 2), np.float32)
    n = C.c_int()
    check(lib.mdc_marker_candidates(mask.ctypes.data, w, h, out.ctypes.data_as(_f32p), capacity, C.byref(n)), "mdc_marker_candidates")
    return out[:n.value].copy()


def marker_read_patch(grey: np.ndarray, quad):
    """The id reader on one quad (mdc_marker_read_patch): (warped 56x56 uint8 patch before Otsu, Otsu threshold, id or -1, rotations)."""
    grey = _u8_image(grey, "grey")
    h, w = grey.shape
    q = np.ascontiguousarray(np.asarray(quad, np.float32).reshape(8))
    patch = np.empty((56, 56), np.uint8)
    t, i, r = C.c_int(), C.c_int(), C.c_int()
    check(lib.mdc_marker_read_patch(grey.ctypes.data, w, h, q.ctypes.data_as(_f32p), patch.ctypes.data, C.byref(t), C.byref(i), C.byref(r)),
          "mdc_marker_read_patch")
    return patch, t.value, i.value, r.value
