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
    ("blinky_build_info", c_char_p, [_CTX]),
    ("blinky_plan_digest", ctypes.c_uint64, [_CTX, c_int]),
    ("blinky_get_tile_plan", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, POINTER(c_size_t), POINTER(c_size_t)]),
    ("blinky_compile_lens", c_int, [_CTX, c_int, POINTER(c_size_t)]),
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
    ("blinky_lens_source", c_int, [_CTX, c_int, c_void_p, c_size_t]),
    ("blinky_write_config", c_int, [_CTX, c_void_p, c_size_t]),
    ("blinky_saveglobe_pending", c_int, [_CTX]),
    ("blinky_save_globe", c_int, [_CTX, c_void_p, c_char_p]),
    ("blinky_set_kernel", c_int, [_CTX, c_int]),
    ("blinky_set_background", c_int, [_CTX, c_void_p]),
    ("blinky_warp_device", c_int, [_CTX, c_void_p, c_size_t, c_void_p, c_size_t, c_int, c_void_p]),
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
    path = os.environ.get("BLINKY_B200_LIB", LIB_PATH)  # (developer builds: make lab)
    if not os.path.exists(path):
        raise ImportError(
            f"{LIB_PATH} is missing: build the CUDA extension first (make -C blinky_b200, or "
            f"__graft_entry__.build()).  blinky_b200 has no CPU fallback for the warp."
        )
    lib = ctypes.CDLL(path)
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

    def lens_source(self, cuda: bool = False, forward: bool = False, with_kernel: bool = False) -> str:
        """The current ``lens_inverse`` (or ``lens_forward``) translated to C++/CUDA (raises when not translatable);
        ``with_kernel`` appends the fixed kernel the device builder launches."""
        flavour = int(cuda) | (2 if forward else 0) | (4 if with_kernel else 0)
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

    def warp(self, d_faces, d_out, nframes: int = 1, face_stride: int | None = None, out_stride: int | None = None,
             stream: int | None = None, rgba: bool = False):
        """device-resident batch; d_faces/d_out are torch CUDA tensors (or raw device addresses)."""
        ps2 = self.platesize * self.platesize
        if face_stride is None:
            face_stride = self.numplates * ps2
        if out_stride is None:
            out_stride = self.width * self.height * (4 if rgba else 1)
        fn = self._lib.blinky_warp_device_rgba if rgba else self._lib.blinky_warp_device
        self._check(fn(self._ctx, _ptr(d_faces), face_stride, _ptr(d_out), out_stride, nframes, stream))

    def warp_host(self, faces: np.ndarray, dst: np.ndarray | None = None, keep_unmapped: bool = False, x0: int = 0,
                  y0: int = 0, nframes: int | None = None, dst_rowbytes: int | None = None,
                  face_stride: int | None = None, dst_frame_stride: int | None = None) -> np.ndarray:
        """end to end from host buffers (numpy uint8, or raw addresses of pinned memory)."""
        ps2 = self.platesize * self.platesize
        if face_stride is None:
            face_stride = self.numplates * ps2
        if nframes is None:
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
