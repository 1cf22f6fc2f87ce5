"""blinky_b200 — H100-native Blinky lens warp (globe faces -> lensmap gather -> screen).

Python host-side mirror of the C ABI in ``include/blinky_b200.h``.  The product
is the C-ABI shared library ``libblinky_b200.so`` (hand-written sm_90a CUDA
kernels + the host-side lensmap builder); this module only binds it with
``ctypes`` so tests and ``bench.py`` can drive it.  There is NO fallback: if the
library is missing or a GPU entry point is called on a host-only context the
call raises.

Reference surface mirrored (all in the reference's engine/NQ/fisheye.c):
console commands (:651-665) via :meth:`Fisheye.command`, ``F_WriteConfig``
(:683-696) via :meth:`Fisheye.write_config`, the lensmap rebuild (:730-743,
:2367-2397) via :meth:`Fisheye.build_lensmap`, and ``render_lensmap``
(:2406-2424) via :meth:`Fisheye.warp` / :meth:`Fisheye.warp_host`.
"""
from __future__ import annotations

import ctypes
import os
import sys
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint8, c_uint32, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libblinky_b200.so")
SCRIPT_DIR = _HERE  # contains lua-scripts/{globes,lenses}

OK = 0
E_INVALID, E_SCRIPT, E_ZOOM, E_NODEVICE, E_CUDA, E_NOMEM, E_STATE = -1, -2, -3, -4, -5, -6, -7
ZOOM_NONE, ZOOM_FOV, ZOOM_VFOV, ZOOM_COVER, ZOOM_CONTAIN = range(5)
MAP_NONE, MAP_INVERSE, MAP_FORWARD = range(3)
MAX_PLATES = 6
LM_VALID = 0x80000000
LM_TINT_SHIFT = 28
LM_TINT_NONE = 7
LM_INDEX_MASK = 0x0FFFFFFF

# every symbol include/blinky_b200.h declares: (name, restype, argtypes)
_CTX = c_void_p
_SIGNATURES = [
    ("blinky_create", c_int, [c_int, POINTER(_CTX)]),
    ("blinky_destroy", None, [_CTX]),
    ("blinky_last_error", c_char_p, [_CTX]),
    ("blinky_version", c_char_p, []),
    ("blinky_set_print_callback", None, [_CTX, c_void_p, c_void_p]),
    ("blinky_set_exec_callback", None, [_CTX, c_void_p, c_void_p]),
    ("blinky_log", c_char_p, [_CTX]),
    ("blinky_log_clear", None, [_CTX]),
    ("blinky_set_basedir", c_int, [_CTX, c_char_p]),
    ("blinky_set_palette", c_int, [_CTX, c_void_p]),
    ("blinky_command", c_int, [_CTX, c_char_p]),
    ("blinky_load_globe", c_int, [_CTX, c_char_p]),
    ("blinky_load_lens", c_int, [_CTX, c_char_p]),
    ("blinky_load_globe_source", c_int, [_CTX, c_char_p, c_char_p]),
    ("blinky_load_lens_source", c_int, [_CTX, c_char_p, c_char_p]),
    ("blinky_set_zoom", c_int, [_CTX, c_int, c_int]),
    ("blinky_set_rubix", c_int, [_CTX, c_int]),
    ("blinky_set_rubixgrid", c_int, [_CTX, c_int, c_double, c_double]),
    ("blinky_build_lensmap", c_int, [_CTX, c_int, c_int, c_int, c_int]),
    ("blinky_needs_rebuild", c_int, [_CTX, c_int, c_int, c_int]),
    ("blinky_set_lensmap", c_int, [_CTX, c_int, c_int, c_int, c_int, c_void_p]),
    ("blinky_set_lensmap_device", c_int, [_CTX, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    ("blinky_set_raymap", c_int, [_CTX, c_int, c_int, c_int, c_void_p]),
    ("blinky_set_raymap_device", c_int, [_CTX, c_int, c_int, c_int, c_void_p, c_void_p]),
    ("blinky_get_raymap", c_int, [_CTX, c_int, c_int, c_void_p]),
    ("blinky_get_raymap_device", c_int, [_CTX, c_int, c_int, c_void_p, c_void_p]),
    ("blinky_get_raymap_forward", c_int, [_CTX, c_int, c_int, c_int, c_void_p]),
    ("blinky_get_raymap_forward_device", c_int, [_CTX, c_int, c_int, c_int, c_void_p, c_void_p]),
    ("blinky_build_info", c_char_p, [_CTX]),
    ("blinky_plan_digest", ctypes.c_uint64, [_CTX, c_int]),
    ("blinky_get_tile_plan", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, POINTER(c_size_t), POINTER(c_size_t)]),
    ("blinky_compile_lens", c_int, [_CTX, c_int, POINTER(c_size_t)]),
    ("blinky_probe_math", c_int, [_CTX, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    ("blinky_fisheye_enabled", c_int, [_CTX]),
    ("blinky_lens_valid", c_int, [_CTX]),
    ("blinky_globe_valid", c_int, [_CTX]),
    ("blinky_lens_name", c_char_p, [_CTX]),
    ("blinky_globe_name", c_char_p, [_CTX]),
    ("blinky_lens_onload", c_char_p, [_CTX]),
    ("blinky_map_type", c_int, [_CTX]),
    ("blinky_zoom_type", c_int, [_CTX]),
    ("blinky_zoom_fov", c_int, [_CTX]),
    ("blinky_max_fov", c_int, [_CTX]),
    ("blinky_max_vfov", c_int, [_CTX]),
    ("blinky_lens_width", c_double, [_CTX]),
    ("blinky_lens_height", c_double, [_CTX]),
    ("blinky_scale", c_double, [_CTX]),
    ("blinky_rubix_enabled", c_int, [_CTX]),
    ("blinky_numplates", c_int, [_CTX]),
    ("blinky_platesize", c_int, [_CTX]),
    ("blinky_width", c_int, [_CTX]),
    ("blinky_height", c_int, [_CTX]),
    ("blinky_get_plates", c_int, [_CTX, c_void_p, c_int]),
    ("blinky_get_display", c_int, [_CTX, c_void_p]),
    ("blinky_plate_fov", c_double, [_CTX, c_int]),
    ("blinky_get_palmaps", c_int, [_CTX, c_void_p]),
    ("blinky_get_lensmap", c_int, [_CTX, c_void_p, c_void_p]),
    ("blinky_get_lensmap_packed", c_int, [_CTX, c_void_p]),
    ("blinky_mapped_pixels", c_int64, [_CTX]),
    ("blinky_lens_inverse", c_int, [_CTX, c_double, c_double, POINTER(c_double)]),
    ("blinky_lens_forward", c_int, [_CTX, c_double, c_double, c_double, POINTER(c_double), POINTER(c_double)]),
    ("blinky_globe_plate", c_int, [_CTX, c_double, c_double, c_double, POINTER(c_int)]),
    ("blinky_lens_source", c_int, [_CTX, c_int, c_void_p, c_size_t]),
    ("blinky_write_config", c_int, [_CTX, c_void_p, c_size_t]),
    ("blinky_saveglobe_pending", c_int, [_CTX]),
    ("blinky_save_globe", c_int, [_CTX, c_void_p, c_char_p]),
    ("blinky_set_kernel", c_int, [_CTX, c_int]),
    ("blinky_set_background", c_int, [_CTX, c_void_p]),
    ("blinky_set_face_layout", c_int, [_CTX, c_int, c_void_p, c_int]),
    ("blinky_warp_device", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_void_p]),
    ("blinky_warp_device_view", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    ("blinky_warp_device_view_rgba", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    ("blinky_warp_device_view_rgba_tables", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_int, c_int, c_int, c_int,
                                                    c_void_p, c_size_t, c_void_p]),
    ("blinky_warp_device_rays", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_int, c_int,
                                        c_int, c_int, c_void_p]),
    ("blinky_warp_device_rays_rgba", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_int,
                                             c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    ("blinky_warp_device_rays_supersampled", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_void_p, c_size_t,
                                                     c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    ("blinky_warp_device_rays_bilinear", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_void_p, c_size_t,
                                                 c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    ("blinky_ray_pyramid_bytes", c_int, [_CTX, POINTER(c_size_t)]),
    ("blinky_warp_device_rays_trilinear", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_size_t, c_int,
                                                  c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p]),
    ("blinky_warp_host", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_int, c_int, c_int, c_int]),
    ("blinky_upload_bytes_per_frame", c_int64, [_CTX]),
    ("blinky_alloc_pinned", c_int, [_CTX, c_size_t, POINTER(c_void_p)]),
    ("blinky_free_pinned", c_int, [_CTX, c_void_p]),
    ("blinky_alloc_device", c_int, [_CTX, c_size_t, POINTER(c_void_p)]),
    ("blinky_free_device", c_int, [_CTX, c_void_p]),
    ("blinky_ipc_export", c_int, [_CTX, c_void_p, c_void_p]),
    ("blinky_ipc_open", c_int, [_CTX, c_void_p, POINTER(c_void_p)]),
    ("blinky_ipc_close", c_int, [_CTX, c_void_p]),
    ("blinky_sync", c_int, [_CTX]),
    ("blinky_release_captures", c_int, [_CTX]),
    ("blinky_set_rgba_table", c_int, [_CTX, c_void_p]),
    ("blinky_warp_device_rgba", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_void_p]),
    ("blinky_plan_summary", c_char_p, [_CTX]),
    ("blinky_launch_count", c_int64, [_CTX]),
    ("blinky_last_kernel", c_char_p, [_CTX]),
    ("blinky_shard_range", c_int, [c_int, c_int, c_int, POINTER(c_int), POINTER(c_int)]),
    ("blinky_shard_unique_id", c_int, [c_void_p]),
    ("blinky_shard_init", c_int, [_CTX, c_int, c_int, c_void_p]),
    ("blinky_shard_buffer", c_int, [_CTX, c_int, POINTER(c_void_p)]),
    ("blinky_shard_warp_gather", c_int, [_CTX, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    ("blinky_shard_sync", c_int, [_CTX]),
    ("blinky_shard_close", c_int, [_CTX]),
]
EXPORTED_SYMBOLS = [s[0] for s in _SIGNATURES]


class BlinkyError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"blinky_b200 error {code}: {message}")
        self.code = code


_lib = None


def load_library() -> ctypes.CDLL:
    """Loads libblinky_b200.so and binds every declared symbol.  Raises if the
    library has not been built (``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build the CUDA extension first (make -C blinky_b200, or "
            f"__graft_entry__.build()).  blinky_b200 has no CPU fallback for the warp."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, restype, argtypes in _SIGNATURES:
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def _ptr(a) -> int:
    """address of a numpy array / torch tensor / int"""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(f"cannot take the address of {type(a)}")


def _warp_stream(stream):
    """stream=None is CUDA's legacy default stream, which cannot be captured: while torch captures on its current
    stream (torch.cuda.graph), a warp goes to that stream instead"""
    if stream is None:
        torch = sys.modules.get("torch")
        if torch is not None and torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing():
            return torch.cuda.current_stream().cuda_stream
    return stream


class Fisheye:
    """One lens-warp context (one per GPU / host thread).

    ``device=None`` makes a host-only context: scripts, console commands and the
    lensmap build work, every warp call raises (code E_NODEVICE).
    """

    def __init__(self, device: int | None = 0, basedir: str | None = None, palette: np.ndarray | None = None):
        self._lib = load_library()
        ctx = _CTX()
        rc = self._lib.blinky_create(-1 if device is None else int(device), ctypes.byref(ctx))
        self._ctx = ctx
        if rc != OK:
            msg = self._lib.blinky_last_error(ctx).decode() if ctx else "out of memory"
            if ctx:
                self._lib.blinky_destroy(ctx)
            self._ctx = None
            raise BlinkyError(rc, msg)
        self.device = device
        self._layout = None   # set_face_layout: (rowbytes, origins) or None for dense faces
        self._lib.blinky_set_basedir(self._ctx, (basedir or SCRIPT_DIR).encode())
        if palette is not None:
            self.set_palette(palette)

    # -- lifecycle -----------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.blinky_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, rc: int):
        if rc != OK:
            raise BlinkyError(rc, self._lib.blinky_last_error(self._ctx).decode())

    # -- configuration ---------------------------------------------------------
    def set_basedir(self, path: str):
        self._check(self._lib.blinky_set_basedir(self._ctx, path.encode()))

    def set_palette(self, palette: np.ndarray):
        pal = np.ascontiguousarray(palette, dtype=np.uint8).reshape(768)
        self._check(self._lib.blinky_set_palette(self._ctx, pal.ctypes.data))

    def command(self, text: str):
        """console surface: 'f_lens panini', 'f_fov 170', 'f_globe cube', 'f_rubix', ..."""
        self._check(self._lib.blinky_command(self._ctx, text.encode()))

    def load_globe(self, name: str, source: str | None = None):
        if source is None:
            self._check(self._lib.blinky_load_globe(self._ctx, name.encode()))
        else:
            self._check(self._lib.blinky_load_globe_source(self._ctx, name.encode(), source.encode()))

    def load_lens(self, name: str, source: str | None = None):
        if source is None:
            self._check(self._lib.blinky_load_lens(self._ctx, name.encode()))
        else:
            self._check(self._lib.blinky_load_lens_source(self._ctx, name.encode(), source.encode()))

    def set_zoom(self, zoom_type: int, fov: int = 0):
        self._check(self._lib.blinky_set_zoom(self._ctx, zoom_type, fov))

    def set_rubix(self, enabled: bool):
        self._check(self._lib.blinky_set_rubix(self._ctx, 1 if enabled else 0))

    def set_rubixgrid(self, numcells: int, cell: float, pad: float):
        self._check(self._lib.blinky_set_rubixgrid(self._ctx, numcells, cell, pad))

    def build_lensmap(self, width: int, height: int, platesize: int = 0, threads: int = 1):
        self._check(self._lib.blinky_build_lensmap(self._ctx, width, height, platesize, threads))

    def set_lensmap(self, packed, platesize: int, numplates: int, stream: int | None = None):
        """Replaces the lensmap with a caller's map of packed entries (LM_* format), [H, W] 32-bit: a numpy array
        (blinky_set_lensmap) or a CUDA tensor (blinky_set_lensmap_device, read on `stream` after the work already
        there, and planned on the GPU).  Rows must be dense."""
        if isinstance(packed, np.ndarray):
            m = np.ascontiguousarray(packed)
            if m.ndim != 2 or m.dtype.itemsize != 4 or m.dtype.kind not in "ui":
                raise ValueError(f"set_lensmap: expected a [H, W] array of 32-bit entries, got {m.dtype} {m.shape}")
            self._check(self._lib.blinky_set_lensmap(self._ctx, m.shape[1], m.shape[0], platesize, numplates, m.ctypes.data))
            return
        if not (hasattr(packed, "is_cuda") and packed.is_cuda):
            raise TypeError("set_lensmap: expected a numpy array or a CUDA tensor")
        if packed.dim() != 2 or packed.element_size() != 4 or not packed.is_contiguous():
            raise ValueError(f"set_lensmap: expected a contiguous [H, W] tensor of 32-bit entries, got {packed.dtype} {tuple(packed.shape)}")
        self._check(self._lib.blinky_set_lensmap_device(self._ctx, packed.shape[1], packed.shape[0], platesize, numplates,
                                                        packed.data_ptr(), stream))

    def set_raymap(self, rays, platesize: int = 0, stream: int | None = None):
        """Maps a view ray per screen pixel through the current globe and installs the result as the lensmap.  rays:
        [H, W, 3] float32, lens_inverse's result narrowed to float and not normalised (the zero vector for an empty
        pixel) — a numpy array (blinky_set_raymap) or a contiguous CUDA tensor (blinky_set_raymap_device, read on
        `stream` after the work already there, mapped and planned on the GPU)."""
        if isinstance(rays, np.ndarray):
            r = np.ascontiguousarray(rays)
            if r.ndim != 3 or r.shape[2] != 3 or r.dtype != np.float32:
                raise ValueError(f"set_raymap: expected a [H, W, 3] float32 array, got {r.dtype} {r.shape}")
            self._check(self._lib.blinky_set_raymap(self._ctx, r.shape[1], r.shape[0], platesize, r.ctypes.data))
            return
        if not (hasattr(rays, "is_cuda") and rays.is_cuda):
            raise TypeError("set_raymap: expected a numpy array or a CUDA tensor")
        if rays.dim() != 3 or rays.shape[2] != 3 or str(rays.dtype) != "torch.float32" or not rays.is_contiguous():
            raise ValueError(f"set_raymap: expected a contiguous [H, W, 3] float32 tensor, got {rays.dtype} {tuple(rays.shape)}")
        self._check(self._lib.blinky_set_raymap_device(self._ctx, rays.shape[1], rays.shape[0], platesize, rays.data_ptr(), stream))

    def raymap(self, width: int, height: int, out=None, stream: int | None = None, *, forward: bool = False, platesize: int = 0):
        """The view rays a width x height build of the current lens evaluates, as set_raymap reads them: [height,
        width, 3] float32, lens_inverse at ((lx - width//2) * scale, -(ly - height//2) * scale) narrowed to float and not
        normalised, the zero vector for nil.  No `out`: a new numpy array (blinky_get_raymap, on the worker threads).
        `out`, a contiguous CUDA float32 [height, width, 3] tensor: filled on `stream` after the work already there
        (blinky_get_raymap_device, evaluated on the GPU) and returned once complete.
        forward=True: the rays of the forward build at width x height on plates of `platesize` texels (0: min(width,
        height)), interpolated through each pixel's winning quad and normalised (blinky_get_raymap_forward[_device],
        DESIGN §3h), for any lens with a lens_forward function; platesize is ignored without it."""
        if out is None:
            rays = np.empty((height, width, 3), np.float32)
            if forward:
                self._check(self._lib.blinky_get_raymap_forward(self._ctx, width, height, platesize, rays.ctypes.data))
            else:
                self._check(self._lib.blinky_get_raymap(self._ctx, width, height, rays.ctypes.data))
            return rays
        if not (hasattr(out, "is_cuda") and out.is_cuda):
            raise TypeError("raymap: out must be a CUDA tensor")
        if tuple(out.shape) != (height, width, 3) or str(out.dtype) != "torch.float32" or not out.is_contiguous():
            raise ValueError(f"raymap: expected a contiguous [{height}, {width}, 3] float32 tensor, got {out.dtype} {tuple(out.shape)}")
        if forward:
            self._check(self._lib.blinky_get_raymap_forward_device(self._ctx, width, height, platesize, out.data_ptr(), stream))
        else:
            self._check(self._lib.blinky_get_raymap_device(self._ctx, width, height, out.data_ptr(), stream))
        return out

    @property
    def build_info(self) -> str:
        """How the last lensmap was built ("device: ..." or "host ...")."""
        return self._lib.blinky_build_info(self._ctx).decode()

    TILE_DTYPE = np.dtype([("entry_offset", "<u4"), ("box_x", "<i2"), ("box_y", "<i2"), ("plate", "u1"), ("type", "u1"),
                           ("box_w16", "u1"), ("box_h8", "u1"), ("px", "<u2"), ("py", "<u2")])

    def tile_plan(self) -> tuple[np.ndarray, np.ndarray]:
        """(tile descriptors as a structured array, entry bytes) exactly as uploaded to the device"""
        nt, nb = c_size_t(), c_size_t()
        self._check(self._lib.blinky_get_tile_plan(self._ctx, None, 0, None, 0, ctypes.byref(nt), ctypes.byref(nb)))
        tiles = np.zeros(nt.value, self.TILE_DTYPE)
        entries = np.zeros(nb.value, np.uint8)
        self._check(self._lib.blinky_get_tile_plan(self._ctx, tiles.ctypes.data, tiles.nbytes, entries.ctypes.data, entries.nbytes, None, None))
        return tiles, entries

    def plan_digest(self, threads: int = 1) -> int:
        return int(self._lib.blinky_plan_digest(self._ctx, threads))

    def compile_lens(self, forward: bool = False) -> int:
        """Translate the current lens to CUDA and compile it with NVRTC; returns the cubin size."""
        n = c_size_t()
        self._check(self._lib.blinky_compile_lens(self._ctx, int(forward), ctypes.byref(n)))
        return n.value

    # blinky_probe_math's ops, in BLINKY_PROBE_* order
    PROBE_OPS = ("sin", "cos", "tan", "asin", "acos", "atan", "atan2", "exp", "log", "log10", "logb", "sinh", "cosh", "tanh", "pow",
                 "sqrt", "fmod", "floor", "ceil", "trunc", "modf", "div", "f32", "int")
    PROBE_BINARY = ("atan2", "logb", "pow", "fmod", "div")

    def probe_math(self, op: str, a=None, b=None, stream: int | None = None):
        """Test hook (blinky_probe_math): the translated lenses' wrapper for `op` (a PROBE_OPS name) on the GPU, as every
        lens unit compiles it.  a, b: contiguous CUDA float64 tensors of one length (b only for PROBE_BINARY ops).
        Returns (value, bound) as new CUDA float64 tensors, complete on return; modf gives (fractional part, integral
        part).  a=None only compiles the unit (works without a GPU)."""
        code = self.PROBE_OPS.index(op)
        if a is None:
            self._check(self._lib.blinky_probe_math(self._ctx, code, None, None, None, None, 0, None))
            return None
        import torch
        for t in (a,) + ((b,) if op in self.PROBE_BINARY else ()):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.is_contiguous() and t.shape == a.shape):
                raise ValueError("probe_math: expected contiguous CUDA float64 tensors of one shape")
        v, e = torch.empty_like(a), torch.empty_like(a)
        if a.numel():
            self._check(self._lib.blinky_probe_math(self._ctx, code, a.data_ptr(), b.data_ptr() if op in self.PROBE_BINARY else None,
                                                    v.data_ptr(), e.data_ptr(), a.numel(), stream))
        return v, e

    def needs_rebuild(self, width: int, height: int, platesize: int = 0) -> bool:
        return bool(self._lib.blinky_needs_rebuild(self._ctx, width, height, platesize))

    # -- queries -----------------------------------------------------------------
    @property
    def log(self) -> str:
        return self._lib.blinky_log(self._ctx).decode(errors="replace")

    def clear_log(self):
        self._lib.blinky_log_clear(self._ctx)

    fisheye_enabled = property(lambda s: bool(s._lib.blinky_fisheye_enabled(s._ctx)))
    lens_valid = property(lambda s: bool(s._lib.blinky_lens_valid(s._ctx)))
    globe_valid = property(lambda s: bool(s._lib.blinky_globe_valid(s._ctx)))
    lens_name = property(lambda s: s._lib.blinky_lens_name(s._ctx).decode())
    globe_name = property(lambda s: s._lib.blinky_globe_name(s._ctx).decode())
    onload = property(lambda s: s._lib.blinky_lens_onload(s._ctx).decode())
    map_type = property(lambda s: s._lib.blinky_map_type(s._ctx))
    zoom_type = property(lambda s: s._lib.blinky_zoom_type(s._ctx))
    zoom_fov = property(lambda s: s._lib.blinky_zoom_fov(s._ctx))
    max_fov = property(lambda s: s._lib.blinky_max_fov(s._ctx))
    max_vfov = property(lambda s: s._lib.blinky_max_vfov(s._ctx))
    lens_width = property(lambda s: s._lib.blinky_lens_width(s._ctx))
    lens_height = property(lambda s: s._lib.blinky_lens_height(s._ctx))
    scale = property(lambda s: s._lib.blinky_scale(s._ctx))
    rubix_enabled = property(lambda s: bool(s._lib.blinky_rubix_enabled(s._ctx)))
    numplates = property(lambda s: s._lib.blinky_numplates(s._ctx))
    platesize = property(lambda s: s._lib.blinky_platesize(s._ctx))
    width = property(lambda s: s._lib.blinky_width(s._ctx))
    height = property(lambda s: s._lib.blinky_height(s._ctx))
    mapped_pixels = property(lambda s: int(s._lib.blinky_mapped_pixels(s._ctx)))
    launch_count = property(lambda s: int(s._lib.blinky_launch_count(s._ctx)))
    last_kernel = property(lambda s: s._lib.blinky_last_kernel(s._ctx).decode())
    upload_bytes_per_frame = property(lambda s: int(s._lib.blinky_upload_bytes_per_frame(s._ctx)))
    plan_summary = property(lambda s: s._lib.blinky_plan_summary(s._ctx).decode())

    def plates(self) -> np.ndarray:
        out = np.zeros((MAX_PLATES, 11), np.float32)
        n = self._lib.blinky_get_plates(self._ctx, out.ctypes.data, MAX_PLATES)
        return out[:n]

    def display(self) -> list[int]:
        out = (c_int * MAX_PLATES)()
        self._lib.blinky_get_display(self._ctx, ctypes.addressof(out))
        return list(out)

    def plate_fov(self, plate: int) -> float:
        return self._lib.blinky_plate_fov(self._ctx, plate)

    def palmaps(self) -> np.ndarray:
        out = np.zeros((MAX_PLATES, 256), np.uint8)
        self._lib.blinky_get_palmaps(self._ctx, out.ctypes.data)
        return out

    def lensmap(self) -> tuple[np.ndarray, np.ndarray]:
        """(idx int32 [H,W] with -1 = unmapped, tint uint8 [H,W] with 255 = none)"""
        h, w = self.height, self.width
        idx = np.empty((h, w), np.int32)
        tint = np.empty((h, w), np.uint8)
        self._check(self._lib.blinky_get_lensmap(self._ctx, idx.ctypes.data, tint.ctypes.data))
        return idx, tint

    def lensmap_packed(self) -> np.ndarray:
        out = np.empty((self.height, self.width), np.uint32)
        self._check(self._lib.blinky_get_lensmap_packed(self._ctx, out.ctypes.data))
        return out

    def lens_inverse(self, x: float, y: float):
        out = (c_double * 3)()
        st = self._lib.blinky_lens_inverse(self._ctx, x, y, out)
        return st, (out[0], out[1], out[2])

    def lens_forward(self, rx: float, ry: float, rz: float):
        x, y = c_double(), c_double()
        st = self._lib.blinky_lens_forward(self._ctx, rx, ry, rz, ctypes.byref(x), ctypes.byref(y))
        return st, (x.value, y.value)

    def globe_plate(self, x: float, y: float, z: float):
        """(status, plate) of the globe's globe_plate script as the lensmap build reads it: status 1 with the plate
        (last value returned, converted like lua_tointeger), 0 with -1 for no value / nil / not a number, negative
        for an error (-2: the globe has no globe_plate, -3: script error)"""
        plate = c_int()
        st = self._lib.blinky_globe_plate(self._ctx, x, y, z, ctypes.byref(plate))
        return st, plate.value

    def lens_source(self, cuda: bool = False, forward: bool = False, with_kernel: bool = False, globe_plate: bool = False,
                    raymap: bool = False, rays: bool = False) -> str:
        """The current ``lens_inverse`` (or ``lens_forward``) translated to C++/CUDA (raises when not translatable);
        ``with_kernel`` appends the fixed kernel the device builder launches and translates the globe's
        ``globe_plate`` into the same unit when there is one.  ``globe_plate``: that function translated alone.
        ``raymap``: the unit of the ray-map kernel (set_raymap on a CUDA tensor), globe_plate and kernel.
        ``rays``: the unit of the ray-export kernel (raymap into a CUDA tensor), lens_inverse and kernel."""
        flavour = (int(cuda) | (2 if forward else 0) | (4 if with_kernel else 0) | (8 if globe_plate else 0) | (16 if raymap else 0)
                   | (32 if rays else 0))
        n = self._lib.blinky_lens_source(self._ctx, flavour, None, 0)
        if n < 0:
            self._check(n)
        buf = ctypes.create_string_buffer(n + 1)
        self._lib.blinky_lens_source(self._ctx, flavour, ctypes.addressof(buf), n + 1)
        return buf.value.decode()

    def write_config(self) -> str:
        n = self._lib.blinky_write_config(self._ctx, None, 0)
        buf = ctypes.create_string_buffer(n + 1)
        self._lib.blinky_write_config(self._ctx, ctypes.addressof(buf), n + 1)
        return buf.value.decode()

    @property
    def saveglobe_pending(self) -> bool:
        return bool(self._lib.blinky_saveglobe_pending(self._ctx))

    def save_globe(self, faces: np.ndarray, directory: str):
        """faces: one frame, dense [numplates, ps, ps] or, with a face layout, the frame's surface"""
        f = np.ascontiguousarray(faces, dtype=np.uint8)
        self._check(self._lib.blinky_save_globe(self._ctx, f.ctypes.data, directory.encode()))

    # -- hot path (GPU only) --------------------------------------------------------
    def set_kernel(self, variant: int):
        self._check(self._lib.blinky_set_kernel(self._ctx, variant))

    def set_background(self, background: np.ndarray | None):
        if background is None:
            self._check(self._lib.blinky_set_background(self._ctx, None))
        else:
            bg = np.ascontiguousarray(background, dtype=np.uint8)
            assert bg.size == self.width * self.height
            self._check(self._lib.blinky_set_background(self._ctx, bg.ctypes.data))

    def set_face_layout(self, rowbytes: int | None = None, origins=None):
        """Where the plates sit in each frame of the faces (blinky_set_face_layout): rows of ``rowbytes`` bytes,
        plate i at byte x, row y = origins[i].  No arguments (or rowbytes 0) restores the dense [numplates, ps, ps]
        faces.  While a layout is set, warp / warp_view / warp_host take the frame stride of a [N, rows, rowbytes]
        faces tensor or array from its stride(0) (otherwise rows * rowbytes, rows = max(y) + platesize)."""
        if not rowbytes:
            self._check(self._lib.blinky_set_face_layout(self._ctx, 0, None, 0))
            self._layout = None
            return
        org = np.ascontiguousarray(np.asarray(origins, dtype=np.int64).reshape(-1, 2))
        if org.min(initial=0) < np.iinfo(np.int32).min or org.max(initial=0) > np.iinfo(np.int32).max:
            raise ValueError("set_face_layout: origins must fit 32-bit integers")
        org = org.astype(np.int32)
        self._check(self._lib.blinky_set_face_layout(self._ctx, int(rowbytes), org.ctypes.data, len(org)))
        self._layout = (int(rowbytes), [tuple(int(v) for v in o) for o in org])

    @property
    def face_layout(self):
        """(rowbytes, [(x, y), ...]) of the face layout, or None for dense faces"""
        return self._layout

    def _face_stride(self, faces) -> int:
        """the default frame stride of `faces`: dense frames, or the face layout's surfaces"""
        if self._layout is None:
            return self.numplates * self.platesize * self.platesize
        if hasattr(faces, "stride") and callable(faces.stride) and faces.dim() >= 3:
            return faces.stride(0) * faces.element_size()
        if isinstance(faces, np.ndarray) and faces.ndim >= 3:
            return faces.strides[0]
        rowbytes, origins = self._layout
        return (max(y for _, y in origins) + self.platesize) * rowbytes

    def warp(self, d_faces, d_out, nframes: int = 1, face_stride: int | None = None, out_stride: int | None = None,
             stream: int | None = None, rgba: bool = False, tables=None):
        """device-resident batch; d_faces/d_out are torch CUDA tensors (or raw device addresses).  May be captured
        into a CUDA graph (torch.cuda.graph; see release_captures).  tables (RGBA): per-frame palette tables, see
        warp_view."""
        if face_stride is None:
            face_stride = self._face_stride(d_faces)
        if out_stride is None:
            out_stride = self.width * self.height * (4 if rgba else 1)
        if tables is not None:
            # the dense frames are the view at (0, 0) of screens exactly as wide as the view
            self.warp_view(d_faces, _ptr(d_out), x0=0, y0=0, rowbytes=self.width * 4, nframes=nframes, rgba=rgba,
                           face_stride=face_stride, screen_stride=out_stride, stream=stream, tables=tables)
            return
        fn = self._lib.blinky_warp_device_rgba if rgba else self._lib.blinky_warp_device
        self._check(fn(self._ctx, _ptr(d_faces), face_stride, _ptr(d_out), out_stride, nframes, _warp_stream(stream)))

    @staticmethod
    def _table_args(tables, rgba: bool, nframes: int) -> tuple[int, int]:
        """(device address, stride in bytes) of per-frame RGBA tables: a CUDA tensor of 4-byte elements, [256] (one
        table for every frame, stride 0) or [N >= nframes, 256] with a contiguous last dimension"""
        if not rgba:
            raise ValueError("tables: per-frame palette tables need rgba=True")
        if not (hasattr(tables, "is_cuda") and hasattr(tables, "element_size")) or not tables.is_cuda:
            raise ValueError("tables: expected a CUDA tensor")
        if tables.element_size() != 4:
            raise ValueError(f"tables: expected 4-byte elements, got {tables.dtype}")
        if tables.dim() == 1 and tuple(tables.shape) == (256,) and tables.stride(0) == 1:
            return tables.data_ptr(), 0
        if tables.dim() == 2 and tables.shape[1] == 256 and tables.stride(1) == 1 and tables.shape[0] >= nframes:
            return tables.data_ptr(), tables.stride(0) * 4
        raise ValueError(f"tables: expected shape [256] or [N >= {nframes}, 256] with a contiguous last dimension, "
                         f"got {tuple(tables.shape)} with strides {tuple(tables.stride())}")

    def warp_view(self, d_faces, d_screen, x0: int = 0, y0: int = 0, rowbytes: int | None = None, nframes: int = 1,
                  keep_unmapped: bool = False, rgba: bool = False, face_stride: int | None = None,
                  screen_stride: int | None = None, stream: int | None = None, tables=None):
        """device-resident batch into the view rectangle at pixel (x0, y0) of device screens (blinky_warp_device_view).
        d_screen: a torch CUDA tensor [N, SH, SW] (or [SH, SW]), whose row pitch and frame stride give rowbytes and
        screen_stride, or a raw device address.  keep_unmapped: only mapped pixels are written.
        tables (RGBA only, blinky_warp_device_view_rgba_tables): frame f is expanded through tables[f] instead of
        the set_rgba_table table — a CUDA tensor of 4-byte elements, [N >= nframes, 256] with a contiguous last
        dimension, or [256] for one table for every frame.  Read when the launch runs, in stream order."""
        if tables is not None:
            d_tables, table_stride = self._table_args(tables, rgba, nframes)
        if face_stride is None:
            face_stride = self._face_stride(d_faces)
        bpp = 4 if rgba else 1
        shape = getattr(d_screen, "shape", None)
        if rowbytes is None:
            rowbytes = d_screen.stride(-2) * d_screen.element_size() if shape is not None and len(shape) >= 2 else (x0 + self.width) * bpp
        if screen_stride is None:
            screen_stride = (d_screen.stride(-3) * d_screen.element_size() if shape is not None and len(shape) >= 3
                             else (y0 + self.height) * rowbytes)
        if tables is not None:
            self._check(self._lib.blinky_warp_device_view_rgba_tables(
                self._ctx, _ptr(d_faces), face_stride, _ptr(d_screen), screen_stride, rowbytes, x0, y0, nframes,
                1 if keep_unmapped else 0, d_tables, table_stride, _warp_stream(stream)))
            return
        fn = self._lib.blinky_warp_device_view_rgba if rgba else self._lib.blinky_warp_device_view
        self._check(fn(self._ctx, _ptr(d_faces), face_stride, _ptr(d_screen), screen_stride, rowbytes, x0, y0, nframes,
                       1 if keep_unmapped else 0, _warp_stream(stream)))

    def warp_rays(self, d_faces, d_screen, rays, xforms=None, *, x0: int = 0, y0: int = 0, rowbytes: int | None = None,
                  nframes: int | None = None, keep_unmapped: bool = False, rgba: bool = False, tables=None,
                  face_stride: int | None = None, screen_stride: int | None = None, stream: int | None = None, supersample: int = 1,
                  filter: str = "nearest", scratch=None):
        """warp_view with each pixel's texel computed on the GPU from its view ray, turned by a per-frame 3x3 matrix,
        through the current globe (blinky_warp_device_rays[_rgba]): frame f equals set_raymap of the turned field
        followed by a one-frame warp_view, without changing the installed lensmap, whose size and background it uses.
        rays: a CUDA float32 tensor [H, W, 3] (one field for every frame) or [N, H, W, 3] (one per frame); xforms: a
        CUDA float32 tensor [3, 3] or [N, 3, 3] of row-major matrices, or None for the rays as they are.  nframes
        defaults to N of whichever is per-frame (else 1).  The other arguments are warp_view's (tables: RGBA only).
        May be captured into a CUDA graph; a replay reads the rays and matrices as they are then.
        supersample=k (2, 3 or 4; RGBA only, blinky_warp_device_rays_supersampled): rays are a k-fold field [k*H, k*W, 3]
        or [N, k*H, k*W, 3], and each pixel is the rounded mean of the colours of its k x k rays (box filter).
        filter="bilinear" (RGBA only, blinky_warp_device_rays_bilinear, with any supersample): each ray's colour blends
        the four texels around where it lands on its plate instead of taking the nearest one.
        filter="trilinear" (RGBA only, supersample 1, blinky_warp_device_rays_trilinear): each frame's plates are
        averaged into a mip pyramid on the GPU, and each pixel blends bilinear colours of the two levels around how far
        apart its neighbouring rays land.  scratch: a contiguous CUDA tensor of at least nframes * ray_pyramid_bytes()
        bytes, 16-byte aligned, which the pyramids are written to; None allocates one for the call, which a stream
        being captured into a graph cannot do (pass a persistent scratch there)."""
        if isinstance(supersample, bool) or not isinstance(supersample, int):
            raise TypeError(f"warp_rays: supersample must be an int (1, 2, 3 or 4), got {supersample!r}")
        if not 1 <= supersample <= 4:
            raise ValueError(f"warp_rays: supersample must be 1, 2, 3 or 4, got {supersample}")
        if supersample > 1 and not rgba:
            raise ValueError("warp_rays: supersample > 1 needs rgba=True (palette indices cannot be averaged)")
        if filter not in ("nearest", "bilinear", "trilinear"):
            raise ValueError(f"warp_rays: filter must be 'nearest' or 'bilinear' or 'trilinear', got {filter!r}")
        if filter in ("bilinear", "trilinear") and not rgba:
            raise ValueError(f"warp_rays: filter={filter!r} needs rgba=True (palette indices cannot be blended)")
        if filter == "trilinear" and supersample != 1:
            raise ValueError("warp_rays: filter='trilinear' takes one sample per pixel (supersample=1)")
        if scratch is not None and filter != "trilinear":
            raise ValueError("warp_rays: scratch is for filter='trilinear' only")
        if not (hasattr(rays, "is_cuda") and rays.is_cuda):
            raise TypeError("warp_rays: rays must be a CUDA tensor")
        W, H = self.width, self.height
        k = supersample
        if str(rays.dtype) != "torch.float32" or rays.dim() not in (3, 4) or tuple(rays.shape[-3:]) != (k * H, k * W, 3) or \
                tuple(rays.stride()[-3:]) != (3 * k * W, 3, 1):
            raise ValueError(f"warp_rays: rays must be float32 [{k * H}, {k * W}, 3] or [N, {k * H}, {k * W}, 3] with contiguous fields, "
                             f"got {rays.dtype} {tuple(rays.shape)} strides {tuple(rays.stride())}")
        if xforms is not None:
            if not (hasattr(xforms, "is_cuda") and xforms.is_cuda):
                raise TypeError("warp_rays: xforms must be a CUDA tensor")
            if str(xforms.dtype) != "torch.float32" or xforms.dim() not in (2, 3) or tuple(xforms.shape[-2:]) != (3, 3) or \
                    tuple(xforms.stride()[-2:]) != (3, 1):
                raise ValueError(f"warp_rays: xforms must be float32 [3, 3] or [N, 3, 3] with contiguous matrices, got "
                                 f"{xforms.dtype} {tuple(xforms.shape)} strides {tuple(xforms.stride())}")
        per_frame = [t.shape[0] for t in (rays, xforms) if t is not None and t.dim() == (4 if t is rays else 3)]
        if nframes is None:
            nframes = min(per_frame) if per_frame else 1
        if rays.dim() == 4 and rays.shape[0] < nframes:
            raise ValueError(f"warp_rays: {rays.shape[0]} ray fields for {nframes} frames")
        if xforms is not None and xforms.dim() == 3 and xforms.shape[0] < nframes:
            raise ValueError(f"warp_rays: {xforms.shape[0]} matrices for {nframes} frames")
        ray_stride = rays.stride(0) * 4 if rays.dim() == 4 else 0
        d_xforms = None if xforms is None else xforms.data_ptr()
        xform_stride = xforms.stride(0) * 4 if xforms is not None and xforms.dim() == 3 else 0
        d_tables, table_stride = (None, 0) if tables is None else self._table_args(tables, rgba, nframes)
        if face_stride is None:
            face_stride = self._face_stride(d_faces)
        bpp = 4 if rgba else 1
        shape = getattr(d_screen, "shape", None)
        if rowbytes is None:
            rowbytes = d_screen.stride(-2) * d_screen.element_size() if shape is not None and len(shape) >= 2 else (x0 + W) * bpp
        if screen_stride is None:
            screen_stride = (d_screen.stride(-3) * d_screen.element_size() if shape is not None and len(shape) >= 3
                             else (y0 + H) * rowbytes)
        args = (self._ctx, _ptr(d_faces), face_stride, rays.data_ptr(), ray_stride, d_xforms, xform_stride, _ptr(d_screen), screen_stride,
                rowbytes, x0, y0, nframes, 1 if keep_unmapped else 0)
        if filter == "trilinear":
            self._warp_rays_trilinear(args, d_tables, table_stride, scratch, nframes, stream)
        elif filter == "bilinear":
            self._check(self._lib.blinky_warp_device_rays_bilinear(*args[:7], k, *args[7:], d_tables, table_stride, _warp_stream(stream)))
        elif k > 1:
            self._check(self._lib.blinky_warp_device_rays_supersampled(*args[:7], k, *args[7:], d_tables, table_stride, _warp_stream(stream)))
        elif rgba:
            self._check(self._lib.blinky_warp_device_rays_rgba(*args, d_tables, table_stride, _warp_stream(stream)))
        else:
            self._check(self._lib.blinky_warp_device_rays(*args, _warp_stream(stream)))

    def ray_pyramid_bytes(self) -> int:
        """bytes of one frame's mip pyramid for warp_rays(filter="trilinear") (blinky_ray_pyramid_bytes): the installed
        lensmap's plate size and every plate of the current globe"""
        n = ctypes.c_size_t(0)
        self._check(self._lib.blinky_ray_pyramid_bytes(self._ctx, ctypes.byref(n)))
        return n.value

    def _warp_rays_trilinear(self, args, d_tables, table_stride, scratch, nframes, stream):
        """blinky_warp_device_rays_trilinear with warp_rays' arguments; scratch None: a torch buffer for this call"""
        own = None
        if scratch is None:
            import torch

            size = max(nframes, 0) * self.ray_pyramid_bytes()
            if torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing():
                raise ValueError("warp_rays: filter='trilinear' under graph capture needs a persistent scratch tensor (scratch=, "
                                 "at least nframes * ray_pyramid_bytes() bytes); allocating one for the call cannot be captured")
            own = torch.empty(max(size, 1), dtype=torch.uint8, device=f"cuda:{self.device}")
            d_scratch, scratch_bytes = own.data_ptr(), size
        else:
            d_scratch = _ptr(scratch)
            scratch_bytes = scratch.numel() * scratch.element_size() if hasattr(scratch, "numel") else None
            if scratch_bytes is None:
                raise TypeError("warp_rays: scratch must be a CUDA tensor (its size is the scratch_bytes passed on)")
            if hasattr(scratch, "is_contiguous") and not scratch.is_contiguous():
                raise ValueError("warp_rays: scratch must be contiguous")
        stream = _warp_stream(stream)
        self._check(self._lib.blinky_warp_device_rays_trilinear(*args, d_tables, table_stride, d_scratch, scratch_bytes, stream))
        if own is not None:
            import torch

            # the buffer goes back to torch's allocator when this call returns: not to be reused before the warp ran
            own.record_stream(torch.cuda.ExternalStream(stream) if stream else torch.cuda.default_stream(own.device))

    def release_captures(self):
        """No CUDA graph that captured a warp of this context will run again (blinky_release_captures): frees the
        lensmap buffers rebuilds kept for such graphs and returns their work counters.  Synchronises the device."""
        self._check(self._lib.blinky_release_captures(self._ctx))

    def warp_host(self, faces: np.ndarray, dst: np.ndarray | None = None, keep_unmapped: bool = False, x0: int = 0,
                  y0: int = 0, nframes: int | None = None, dst_rowbytes: int | None = None,
                  face_stride: int | None = None, dst_frame_stride: int | None = None) -> np.ndarray:
        """end to end from host buffers (numpy uint8, or raw addresses of pinned memory)."""
        if face_stride is None:
            face_stride = self._face_stride(faces)
        if nframes is None:
            if self._layout is not None and isinstance(faces, np.ndarray) and faces.ndim >= 3:
                nframes = faces.shape[0]
            else:
                nframes = int(faces.size // face_stride) if isinstance(faces, np.ndarray) else 1
        if dst is None:
            dst = np.zeros((nframes, self.height, self.width), np.uint8)
        if dst_rowbytes is None:
            dst_rowbytes = dst.shape[-1] if isinstance(dst, np.ndarray) else self.width
        if dst_frame_stride is None:
            dst_frame_stride = (dst.shape[-1] * dst.shape[-2]) if isinstance(dst, np.ndarray) else self.width * self.height
        self._check(self._lib.blinky_warp_host(self._ctx, _ptr(faces), face_stride, _ptr(dst), dst_frame_stride,
                                               dst_rowbytes, x0, y0, nframes, 1 if keep_unmapped else 0))
        return dst

    def alloc_pinned(self, nbytes: int) -> np.ndarray:
        """pinned host memory as a numpy uint8 array (freed with free_pinned)"""
        p = c_void_p()
        self._check(self._lib.blinky_alloc_pinned(self._ctx, nbytes, ctypes.byref(p)))
        return np.ctypeslib.as_array(ctypes.cast(p, POINTER(c_uint8)), shape=(nbytes,))

    def free_pinned(self, arr: np.ndarray):
        self._check(self._lib.blinky_free_pinned(self._ctx, arr.ctypes.data))

    # -- peer memory (fused warp + gather) -------------------------------------------------
    def alloc_device(self, nbytes: int) -> int:
        p = c_void_p()
        self._check(self._lib.blinky_alloc_device(self._ctx, nbytes, ctypes.byref(p)))
        return p.value

    def free_device(self, ptr: int):
        self._check(self._lib.blinky_free_device(self._ctx, ptr))

    def ipc_export(self, ptr: int) -> bytes:
        h = ctypes.create_string_buffer(64)
        self._check(self._lib.blinky_ipc_export(self._ctx, ptr, ctypes.addressof(h)))
        return h.raw

    def ipc_open(self, handle: bytes) -> int:
        h = ctypes.create_string_buffer(handle, 64)
        p = c_void_p()
        self._check(self._lib.blinky_ipc_open(self._ctx, ctypes.addressof(h), ctypes.byref(p)))
        return p.value

    def ipc_close(self, ptr: int):
        self._check(self._lib.blinky_ipc_close(self._ctx, ptr))

    # -- sharded batches (one process per GPU) ----------------------------------------------
    def shard_init(self, rank: int, world: int, unique_id: bytes):
        buf = ctypes.create_string_buffer(unique_id, 128)
        self._check(self._lib.blinky_shard_init(self._ctx, rank, world, ctypes.addressof(buf)))

    def shard_buffer(self, total_frames: int) -> int | None:
        """collective; rank 0 gets the device address of the gather buffer, the others None"""
        p = c_void_p()
        self._check(self._lib.blinky_shard_buffer(self._ctx, total_frames, ctypes.byref(p)))
        return p.value

    def shard_warp_gather(self, d_faces, total_frames: int, mode: int = 0, chunk_frames: int = 2, face_stride: int | None = None,
                          stream: int | None = None):
        if face_stride is None:
            face_stride = self.numplates * self.platesize * self.platesize
        self._check(self._lib.blinky_shard_warp_gather(self._ctx, _ptr(d_faces), face_stride, total_frames, mode, chunk_frames, stream))

    def shard_sync(self):
        self._check(self._lib.blinky_shard_sync(self._ctx))

    def shard_close(self):
        self._check(self._lib.blinky_shard_close(self._ctx))

    def set_rgba_table(self, table: np.ndarray):
        t = np.ascontiguousarray(table, dtype=np.uint32).reshape(256)
        self._check(self._lib.blinky_set_rgba_table(self._ctx, t.ctypes.data))

    def sync(self):
        self._check(self._lib.blinky_sync(self._ctx))


GATHER_NCCL, GATHER_PEER_COPY, GATHER_PEER_STORE = 0, 1, 2


def shard_range(total_frames: int, rank: int, world: int) -> range:
    """frames owned by `rank` (blinky_shard_range: contiguous blocks, sizes differ by at most one)"""
    first, count = c_int(), c_int()
    rc = load_library().blinky_shard_range(total_frames, rank, world, ctypes.byref(first), ctypes.byref(count))
    if rc != OK:
        raise BlinkyError(rc, "blinky_shard_range: bad arguments")
    return range(first.value, first.value + count.value)


def shard_unique_id() -> bytes:
    """128-byte NCCL id made on one rank and carried to the others by the caller"""
    buf = ctypes.create_string_buffer(128)
    rc = load_library().blinky_shard_unique_id(ctypes.addressof(buf))
    if rc != OK:
        raise BlinkyError(rc, "blinky_shard_unique_id failed (is libnccl.so.2 loadable?)")
    return buf.raw


def usable_cpus() -> int:
    """CPUs this process may really use: the affinity mask capped by the cgroup CPU quota
    (a container can show 128 CPUs and be throttled to 24)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(quota) // int(period)))
    except (OSError, ValueError):
        pass
    return max(1, n)


def synthetic_palette(seed: int = 7) -> np.ndarray:
    """the seeded stand-in for gfx/palette.lmp used by tests and bench (BASELINE.md section 2)"""
    return np.random.default_rng(seed).integers(0, 256, 768, dtype=np.uint8)


def synthetic_faces(numplates: int, platesize: int, frame: int = 0) -> np.ndarray:
    """uint8[P][ps][ps] i.i.d. uniform, seed 1000+frame (SURVEY.md section 8d)"""
    return np.random.default_rng(1000 + frame).integers(0, 256, (numplates, platesize, platesize), dtype=np.uint8)


def synthetic_background(width: int, height: int) -> np.ndarray:
    return np.random.default_rng(3).integers(0, 256, (height, width), dtype=np.uint8)
