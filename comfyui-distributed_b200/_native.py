"""ctypes binding of libusdu_b200.so (C ABI declared in include/usdu_b200.h).

There is no fallback: if the shared library is missing or a call fails, a
``NativeError`` is raised.  The library is built in-tree by ``__graft_entry__.build()``
(``make -C comfyui-distributed_b200/csrc``).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_uint32, c_void_p

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libusdu_b200.so")

# constants mirrored from include/usdu_b200.h (checked against the header in tests)
ABI_VERSION = 19
ERR_INVALID = -1
CANVAS_SLACK = 16
PLAN_INFO_WORDS = 16
(PI_TW, PI_TH, PI_TILES, PI_TAB_WORDS, PI_TABLES, PI_MASK_CLASSES, PI_MASK_POOL_BYTES, PI_FAST, PI_MMA, PI_PATH,
 PI_NEIGHBOR_WORDS) = range(11)
PLAN_TILE_WORDS = 12
PLAN_TABLE_WORDS = 8
WL_INFO_WORDS = 16
(WL_ITEMS, WL_ITEM_WORDS, WL_COVER, WL_PATCH_W, WL_PATCH_H, WL_ALGO_BYTES, WL_N_LAUNCH, WL_BLOCK_ROWS, WL_BLOCK_COLS,
 WL_ROW0, WL_ROW1, WL_PATH, WL_KS2, WL_TOTAL, WL_FLAGS, WL_GRID) = range(16)
TILE_WORDS = 24
T_X1, T_Y1, T_EW, T_EH, T_PW, T_PH, T_MASK_OFF, T_MASK_PITCH = range(8)
T_TAB_CROP_H, T_TAB_CROP_V, T_TAB_BLEND_H, T_TAB_BLEND_V = 8, 9, 10, 11
T_SUP_X0, T_SUP_Y0, T_SUP_X1, T_SUP_Y1 = 12, 13, 14, 15
T_FULL_X0, T_FULL_Y0, T_FULL_X1, T_FULL_Y1 = 16, 17, 18, 19
TAB_HEADER = 8
PACKED_ROW = 8
FLAG_FAST = 1
FLAG_MMA = 2
FLAG_MMA_KS2 = 4
FLAG_REMOTE_CANVAS = 1 << 24
FILTER_LANCZOS, FILTER_BICUBIC = 0, 1
CROP_ITEM_WORDS = 6
BLEND_ITEM_WORDS = 4
COVER_WORDS = 4
MASK_WORDS = 16
BLOCK_W = 64
BLOCK_H = 32
FAST_BLOCK_W = 128
FAST_BLOCK_H = 32
FAST_TAPS = 7
JOB_WORDS = 32
(J_SRC_A, J_SRC_B, J_LEAD, J_COLS, J_ROWS, J_IX0, J_IY0, J_ROWS_H, J_OX_BASE, J_N_OUT_H, J_ROWS_V, J_OY_BASE, J_N_OUT_V,
 J_DST_X, J_DST_Y, J_OFF_LO, J_OFF_HI, J_ROWS_OUT, J_COLS_OUT, J_CX0, J_CX1, J_CY0, J_CY1, J_FLAGS, J_MPITCH, J_PITCH,
 J_FRAME_LO, J_FRAME_HI, J_NEXT, J_TAPS_H, J_TAPS_V) = range(31)


class NativeError(RuntimeError):
    pass


_lib = None

_SIGNATURES = {
    "usdu_abi_version": (c_int, []),
    "usdu_last_error": (c_char_p, []),
    "usdu_device_count": (c_int, []),
    "usdu_sm_count": (c_int, []),
    "usdu_resample_ksize": (c_int, [c_int, c_int]),
    "usdu_resample_table_words": (c_int64, [c_int, c_int]),
    "usdu_build_resample_table": (c_int, [c_int, c_int, POINTER(c_int32)]),
    "usdu_build_identity_table": (c_int, [c_int, POINTER(c_int32)]),
    "usdu_filter_ksize": (c_int, [c_int, c_int, c_int]),
    "usdu_filter_table_words": (c_int64, [c_int, c_int, c_int]),
    "usdu_build_filter_table": (c_int, [c_int, c_int, c_int, POINTER(c_int32)]),
    "usdu_nearest_index": (c_int, [c_int, c_int, POINTER(c_int32)]),
    "usdu_table_input_span": (c_int, [POINTER(c_int32), c_int, c_int, POINTER(c_int), POINTER(c_int)]),
    "usdu_box_blur_params": (c_int, [c_float, POINTER(c_int32), POINTER(c_uint32), POINTER(c_uint32)]),
    "usdu_quantize_canvas": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_void_p]),
    "usdu_dequantize_canvas": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_void_p]),
    "usdu_gather_dequantize": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int64, c_void_p]),
    "usdu_gather_canvas": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int64, c_void_p]),
    "usdu_tile_crop_resize_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "usdu_quantize_rows": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int, c_int, c_void_p]),
    "usdu_dequantize_rows": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int, c_int, c_void_p]),
    "usdu_stream_args_set": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "usdu_quantize_rows_streamed": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int, c_int, c_int, c_void_p]),
    "usdu_dequantize_rows_streamed": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int, c_int, c_int, c_void_p]),
    "usdu_graph_instantiate": (c_int, [c_void_p, c_int, POINTER(c_void_p)]),
    "usdu_graph_launch": (c_int, [c_void_p, c_void_p]),
    "usdu_graph_exec_destroy": (c_int, [c_void_p]),
    "usdu_pack_tiles_u8": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "usdu_unpack_tiles_f32": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "usdu_png_sizes": (c_int, [c_int, c_int, c_int, POINTER(c_int64), POINTER(c_int64), POINTER(c_int64)]),
    "usdu_png_base64_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "usdu_png_decode_u8": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "usdu_png_decode_warps": (c_int, [c_int]),
    "usdu_png_decode_general_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "usdu_jpeg_parse": (c_int, [c_void_p, c_int64, POINTER(c_int64), POINTER(c_int32)]),
    "usdu_jpeg_decode_coefs": (c_int, [c_void_p, c_int64, c_void_p, c_int64]),
    "usdu_jpeg_decode_u8": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "usdu_png_encode_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p, c_int, c_void_p,
                                   c_int, POINTER(c_int64), c_void_p, c_void_p, c_void_p]),
    "usdu_gather_unpack_f32": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "usdu_b64_png_check": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "usdu_t0_denoise": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_float, c_void_p]),
    "usdu_mask_scratch_bytes": (c_int64, [POINTER(c_int32), c_int]),
    "usdu_build_feather_masks": (c_int, [POINTER(c_int32), c_int, c_void_p, c_void_p, c_void_p]),
    "usdu_plane_resample_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int64, c_void_p, c_int, c_int,
                                       c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int64, c_int64,
                                       c_void_p]),
    "usdu_plane_pad_fill_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int64, c_int, c_int, c_void_p,
                                       c_void_p, c_void_p, c_int64, c_int64, c_void_p]),
    "usdu_tile_crop_resize": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p,
                                      c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "usdu_tile_blend": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "usdu_canvas_pitch": (c_int64, [c_int]),
    "usdu_canvas_bytes": (c_int64, [c_int, c_int, c_int]),
    "usdu_plan_create": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_void_p)]),
    "usdu_plan_destroy": (c_int, [c_void_p]),
    "usdu_plan_info": (c_int, [c_void_p, POINTER(c_int64)]),
    "usdu_plan_tiles": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_plan_tile_desc": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_plan_tables": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_plan_table_index": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_plan_mask_specs": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_plan_neighbors": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_int32)]),
    "usdu_plan_waves": (c_int, [c_void_p, POINTER(c_int32), c_int, POINTER(c_int32)]),
    "usdu_plan_crop_worklist": (c_int, [c_void_p, POINTER(c_int32), c_int, c_int, c_int, c_int, c_int, POINTER(c_void_p)]),
    "usdu_plan_blend_worklist": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_int64), c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, POINTER(c_void_p)]),
    "usdu_plan_split_worklists": (c_int, [c_void_p, POINTER(c_int32), POINTER(c_int64), c_int, POINTER(c_int32), c_int, c_int,
                                          c_int, c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p)]),
    "usdu_mma_resident_ctas": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "usdu_worklist_destroy": (c_int, [c_void_p]),
    "usdu_worklist_info": (c_int, [c_void_p, POINTER(c_int64)]),
    "usdu_worklist_items": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_worklist_cover": (c_int, [c_void_p, POINTER(c_int32)]),
    "usdu_worklist_slots": (c_int, [c_void_p, POINTER(c_int64)]),
}

EXPORTS = tuple(_SIGNATURES)


def lib():
    """Load (once) and return the ctypes handle; raises NativeError when absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise NativeError(
            f"{LIB_PATH} not found: the CUDA extension has not been built "
            "(run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C comfyui-distributed_b200/csrc`). "
            "There is no CPU fallback.")
    try:
        h = ctypes.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise NativeError(f"cannot load {LIB_PATH}: {e}") from e
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(h, name)
        except AttributeError as e:
            raise NativeError(f"{LIB_PATH} does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    if h.usdu_abi_version() != ABI_VERSION:
        raise NativeError(f"ABI mismatch: library {h.usdu_abi_version()} != binding {ABI_VERSION}")
    _lib = h
    return h


def _check(status: int, what: str):
    if status != 0:
        msg = lib().usdu_last_error()
        raise NativeError(f"{what} failed ({status}): {msg.decode() if msg else '?'}")


def _i32p(a: np.ndarray):
    assert a.dtype == np.int32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(POINTER(c_int32))


KERNEL_CROP_LDG, KERNEL_CROP_TMA, KERNEL_BLEND, KERNEL_LARGE = 0, 1, 2, 4


def resident_ctas(kernel: int, two_ksteps: bool, patch_w: int, patch_h: int, block_rows: int, use_device: bool) -> int:
    """Resident CTAs per SM of a tensor-core kernel build at the shared memory its launcher requests for these patch
    words (usdu_mma_resident_ctas): the device's occupancy calculator, or the library's table without it."""
    n = lib().usdu_mma_resident_ctas(kernel, int(two_ksteps), patch_w, patch_h, block_rows, int(use_device))
    if n < 0:
        _check(n, "usdu_mma_resident_ctas")
    return n


# ---- host-side builders -------------------------------------------------------------
def sm_count() -> int:
    """SMs of the current CUDA device (the count the launchers size their grids with), or 0 without a device."""
    n = lib().usdu_sm_count()
    return n if n > 0 else 0


def build_resample_table(in_size: int, out_size: int) -> np.ndarray:
    L = lib()
    words = L.usdu_resample_table_words(in_size, out_size)
    if words < 0:
        _check(int(words), "usdu_resample_table_words")
    tab = np.zeros(int(words), dtype=np.int32)
    _check(L.usdu_build_resample_table(in_size, out_size, _i32p(tab)), "usdu_build_resample_table")
    if tab[4]:                                   # trim the packed section to its actual row stride
        tab = tab[: int(tab[4]) + out_size * int(tab[6])]
    return np.ascontiguousarray(tab)


def build_filter_table(filt: int, in_size: int, out_size: int) -> np.ndarray:
    """Generic-kernel table (header + bounds + kk) of a LANCZOS / BICUBIC axis; the packed rows
    of the fast tile kernels are dropped."""
    L = lib()
    words = L.usdu_filter_table_words(filt, in_size, out_size)
    if words < 0:
        _check(int(words), "usdu_filter_table_words")
    tab = np.zeros(int(words), dtype=np.int32)
    _check(L.usdu_build_filter_table(filt, in_size, out_size, _i32p(tab)), "usdu_build_filter_table")
    return np.ascontiguousarray(tab[: TAB_HEADER + out_size * (2 + int(tab[2]))])


def nearest_index(in_size: int, out_size: int) -> np.ndarray:
    idx = np.zeros(out_size, dtype=np.int32)
    _check(lib().usdu_nearest_index(in_size, out_size, _i32p(idx)), "usdu_nearest_index")
    return idx


def table_input_span(table: np.ndarray, first_out: int, n_out: int):
    a, b = c_int(), c_int()
    _check(lib().usdu_table_input_span(_i32p(table), first_out, n_out, ctypes.byref(a), ctypes.byref(b)),
           "usdu_table_input_span")
    return a.value, b.value


def build_identity_table(size: int) -> np.ndarray:
    tab = np.zeros(((TAB_HEADER + 3 * size + 3) & ~3) + size * PACKED_ROW, dtype=np.int32)
    _check(lib().usdu_build_identity_table(size, _i32p(tab)), "usdu_build_identity_table")
    return tab


def box_blur_params(radius: float):
    rad, ww, fw = c_int32(), c_uint32(), c_uint32()
    _check(lib().usdu_box_blur_params(float(radius), ctypes.byref(rad), ctypes.byref(ww), ctypes.byref(fw)),
           "usdu_box_blur_params")
    return rad.value, ww.value, fw.value


def canvas_bytes(B: int, H: int, W: int) -> int:
    n = lib().usdu_canvas_bytes(B, H, W)
    if n < 0:
        _check(int(n), "usdu_canvas_bytes")
    return int(n)


# ---- host-side planner (usdu_plan_*) --------------------------------------------------
def _i64p(a: np.ndarray):
    assert a.dtype == np.int64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(POINTER(c_int64))


def _ids(tile_ids) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(tile_ids, dtype=np.int64).reshape(-1).astype(np.int32))


def _read_worklist(h: c_void_p) -> dict:
    """Contents of a usdu_worklist handle (destroyed here): info words, items int32 [n, words], cover int32 [m, 4]
    and the crop's slot offsets int64."""
    L = lib()
    try:
        info = np.zeros(WL_INFO_WORDS, np.int64)
        _check(L.usdu_worklist_info(h, _i64p(info)), "usdu_worklist_info")
        items = np.zeros((int(info[WL_ITEMS]), int(info[WL_ITEM_WORDS])), np.int32)
        if items.size:
            _check(L.usdu_worklist_items(h, _i32p(items)), "usdu_worklist_items")
        cover = np.zeros((int(info[WL_COVER]), COVER_WORDS), np.int32)
        if cover.size:
            _check(L.usdu_worklist_cover(h, _i32p(cover)), "usdu_worklist_cover")
        return {"info": info, "items": items, "cover": cover}
    finally:
        L.usdu_worklist_destroy(h)


class NativePlan:
    """Owner of one usdu_plan handle: the library's planner for one job geometry (include/usdu_b200.h, planner
    section).  Inputs the library rejects (a tile size that rounds to zero, feather templates of 2 GiB or more ...)
    raise ValueError with the library's message."""

    def __init__(self, W: int, H: int, tile_width: int, tile_height: int, padding: int, mask_blur: int, uniform: bool):
        L = lib()
        self._lib = L
        self._h = c_void_p()
        st = L.usdu_plan_create(W, H, tile_width, tile_height, padding, mask_blur, int(bool(uniform)), ctypes.byref(self._h))
        if st == ERR_INVALID:
            raise ValueError(L.usdu_last_error().decode())
        _check(st, "usdu_plan_create")
        self.info = np.zeros(PLAN_INFO_WORDS, np.int64)
        _check(L.usdu_plan_info(self._h, _i64p(self.info)), "usdu_plan_info")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._lib.usdu_plan_destroy(h)
            self._h = None

    def _array(self, fn: str, shape) -> np.ndarray:
        a = np.zeros(shape, np.int32)
        if a.size:
            _check(getattr(self._lib, fn)(self._h, _i32p(a)), fn)
        return a

    def tiles(self) -> np.ndarray:
        return self._array("usdu_plan_tiles", (int(self.info[PI_TILES]), PLAN_TILE_WORDS))

    def tile_desc(self) -> np.ndarray:
        return self._array("usdu_plan_tile_desc", (int(self.info[PI_TILES]), TILE_WORDS))

    def tables(self) -> np.ndarray:
        return self._array("usdu_plan_tables", int(self.info[PI_TAB_WORDS]))

    def table_index(self) -> np.ndarray:
        return self._array("usdu_plan_table_index", (int(self.info[PI_TABLES]), PLAN_TABLE_WORDS))

    def mask_specs(self) -> np.ndarray:
        return self._array("usdu_plan_mask_specs", (int(self.info[PI_MASK_CLASSES]), MASK_WORDS))

    def neighbors(self):
        T = int(self.info[PI_TILES])
        first = np.zeros(T + 1, np.int32)
        lst = np.zeros(max(int(self.info[PI_NEIGHBOR_WORDS]), 1), np.int32)
        _check(self._lib.usdu_plan_neighbors(self._h, _i32p(first), _i32p(lst)), "usdu_plan_neighbors")
        return [lst[first[i]:first[i + 1]].tolist() for i in range(T)]

    def waves(self, order) -> np.ndarray:
        """Level of every entry of `order` (usdu_plan_waves)."""
        ids = _ids(order)
        level = np.zeros(max(ids.size, 1), np.int32)
        st = self._lib.usdu_plan_waves(self._h, _i32p(ids), ids.size, _i32p(level))
        if st == ERR_INVALID:
            raise ValueError(self._lib.usdu_last_error().decode())
        _check(min(st, 0), "usdu_plan_waves")
        return level[:ids.size]

    def crop_worklist(self, tile_ids, B: int, path: int, sm_count: int, mma_block_rows: int) -> dict:
        ids = _ids(tile_ids)
        h = c_void_p()
        _check(self._lib.usdu_plan_crop_worklist(self._h, _i32p(ids), ids.size, B, path, sm_count, mma_block_rows, ctypes.byref(h)),
               "usdu_plan_crop_worklist")
        slots = np.zeros(max(ids.size, 1), np.int64)
        if ids.size:
            _check(self._lib.usdu_worklist_slots(h, _i64p(slots)), "usdu_worklist_slots")
        out = _read_worklist(h)
        out["slots"] = slots[:ids.size]
        return out

    def split_worklists(self, tile_ids, offs, prev_ids, B: int, path: int, sm_count: int) -> tuple:
        """-> (late crop, early crop, blend) of one wave of the split schedule; the crops carry "slots"."""
        ids, prev = _ids(tile_ids), _ids(prev_ids)
        offs = np.ascontiguousarray(np.asarray(offs, dtype=np.int64).reshape(-1))
        if offs.size < ids.size:
            raise ValueError(f"split work lists: {offs.size} source offsets for {ids.size} tiles")
        offs = np.ascontiguousarray(offs[:max(ids.size, 1)]) if offs.size else np.zeros(1, np.int64)
        hs = [c_void_p() for _ in range(3)]
        _check(self._lib.usdu_plan_split_worklists(self._h, _i32p(ids), _i64p(offs), ids.size, _i32p(prev), prev.size, B, path,
                                                   sm_count, *[ctypes.byref(h) for h in hs]), "usdu_plan_split_worklists")
        slots = np.zeros(max(ids.size, 1), np.int64)
        try:
            if ids.size:
                _check(self._lib.usdu_worklist_slots(hs[0], _i64p(slots)), "usdu_worklist_slots")
        except BaseException:
            for h in hs:
                self._lib.usdu_worklist_destroy(h)
            raise
        out = [_read_worklist(h) for h in hs]
        out[0]["slots"] = out[1]["slots"] = slots[:ids.size]
        return tuple(out)

    def blend_worklist(self, tile_ids, offs, src_bytes: int, B: int, path: int, part, sm_count: int, mma_block_rows: int) -> dict:
        """part = (i, n) or None."""
        ids = _ids(tile_ids)
        offs = np.ascontiguousarray(np.asarray(offs, dtype=np.int64).reshape(-1))
        if offs.size < ids.size:
            raise ValueError(f"blend work list: {offs.size} source offsets for {ids.size} tiles")
        offs = np.ascontiguousarray(offs[:max(ids.size, 1)]) if offs.size else np.zeros(1, np.int64)
        pi, pn = part if part is not None else (0, 0)
        h = c_void_p()
        _check(self._lib.usdu_plan_blend_worklist(self._h, _i32p(ids), _i64p(offs), ids.size, src_bytes, B, path, pi, pn,
                                                  sm_count, mma_block_rows, ctypes.byref(h)), "usdu_plan_blend_worklist")
        return _read_worklist(h)


# ---- device entry points (raw pointers; torch supplies memory and the stream) ----------
def quantize_canvas(img_ptr, canvas_ptr, B, H, W, pitch, stream):
    _check(lib().usdu_quantize_canvas(img_ptr, canvas_ptr, B, H, W, pitch, stream), "usdu_quantize_canvas")


def quantize_rows(img_ptr, canvas_ptr, B, H, W, pitch, y0, y1, stream):
    _check(lib().usdu_quantize_rows(img_ptr, canvas_ptr, B, H, W, pitch, y0, y1, stream), "usdu_quantize_rows")


def dequantize_rows(canvas_ptr, img_ptr, B, H, W, pitch, y0, y1, stream):
    _check(lib().usdu_dequantize_rows(canvas_ptr, img_ptr, B, H, W, pitch, y0, y1, stream), "usdu_dequantize_rows")


STREAM_ARGS_BYTES = 16          # sizeof(usdu_stream_args): the fp32 image and result addresses


def stream_args_set(args_ptr, img_ptr, out_ptr, stream):
    _check(lib().usdu_stream_args_set(args_ptr, img_ptr, out_ptr, stream), "usdu_stream_args_set")


def quantize_rows_streamed(args_ptr, canvas_ptr, B, H, W, pitch, y0, y1, max_ctas, stream):
    _check(lib().usdu_quantize_rows_streamed(args_ptr, canvas_ptr, B, H, W, pitch, y0, y1, max_ctas, stream),
           "usdu_quantize_rows_streamed")


def dequantize_rows_streamed(canvas_ptr, args_ptr, B, H, W, pitch, y0, y1, max_ctas, stream):
    _check(lib().usdu_dequantize_rows_streamed(canvas_ptr, args_ptr, B, H, W, pitch, y0, y1, max_ctas, stream),
           "usdu_dequantize_rows_streamed")


def graph_instantiate(graph_handle: int, high_priority: bool) -> int:
    """cudaGraphExec_t (as an int) of a captured cudaGraph_t; see usdu_graph_instantiate."""
    h = c_void_p()
    _check(lib().usdu_graph_instantiate(graph_handle, int(bool(high_priority)), ctypes.byref(h)), "usdu_graph_instantiate")
    return int(h.value)


def graph_launch(exec_handle: int, stream):
    _check(lib().usdu_graph_launch(exec_handle, stream), "usdu_graph_launch")


def graph_exec_destroy(exec_handle: int):
    _check(lib().usdu_graph_exec_destroy(exec_handle), "usdu_graph_exec_destroy")


def gather_dequantize(slab_ptrs, slab_rows, img_ptr, B, H, W, pitch, stream):
    """slab_ptrs: device addresses of the n canvases; slab_rows: n + 1 row boundaries (0 .. H)."""
    n = len(slab_ptrs)
    ptrs = (ctypes.c_void_p * n)(*[int(p) for p in slab_ptrs])
    rows = (c_int32 * (n + 1))(*[int(r) for r in slab_rows])
    _check(lib().usdu_gather_dequantize(ptrs, rows, n, img_ptr, B, H, W, pitch, stream), "usdu_gather_dequantize")


def gather_canvas(slab_ptrs, slab_rows, canvas_ptr, B, H, W, pitch, stream):
    n = len(slab_ptrs)
    ptrs = (ctypes.c_void_p * n)(*[int(p) for p in slab_ptrs])
    rows = (c_int32 * (n + 1))(*[int(r) for r in slab_rows])
    _check(lib().usdu_gather_canvas(ptrs, rows, n, canvas_ptr, B, H, W, pitch, stream), "usdu_gather_canvas")


def tile_crop_resize_f32(image_ptr, B, H, W, tabs_ptr, items_ptr, n_items, patch_w, patch_h, out_ptr, flags, stream):
    _check(lib().usdu_tile_crop_resize_f32(image_ptr, B, H, W, tabs_ptr, items_ptr, n_items, patch_w, patch_h, out_ptr, flags, stream),
           "usdu_tile_crop_resize_f32")


def dequantize_canvas(canvas_ptr, img_ptr, B, H, W, pitch, stream):
    _check(lib().usdu_dequantize_canvas(canvas_ptr, img_ptr, B, H, W, pitch, stream), "usdu_dequantize_canvas")


def pack_tiles_u8(src_ptr, dst_ptr, n, stream):
    _check(lib().usdu_pack_tiles_u8(src_ptr, dst_ptr, n, stream), "usdu_pack_tiles_u8")


def unpack_tiles_f32(src_ptr, dst_ptr, n, stream):
    _check(lib().usdu_unpack_tiles_f32(src_ptr, dst_ptr, n, stream), "usdu_unpack_tiles_f32")


def png_sizes(H: int, W: int, C: int):
    """-> (PNG bytes, base64 text bytes, device staging bytes) of one [H, W, C] frame (usdu_png_sizes)."""
    png, text, staging = c_int64(), c_int64(), c_int64()
    _check(lib().usdu_png_sizes(H, W, C, ctypes.byref(png), ctypes.byref(text), ctypes.byref(staging)), "usdu_png_sizes")
    return png.value, text.value, staging.value


def png_base64_u8(src_ptr, B, H, W, C, staging_ptr, text_ptr, stream):
    _check(lib().usdu_png_base64_u8(src_ptr, B, H, W, C, staging_ptr, text_ptr, stream), "usdu_png_base64_u8")


PNG_DESC_WORDS = 8
PNG_MAX_ROW_BYTES = 65536      # 16,384 px (ComfyUI's MAX_RESOLUTION) at 4 channels


def png_decode_u8(src_ptr, segs_ptr, n_segs, descs_ptr, n, max_row_bytes, dst_ptr, stream):
    _check(lib().usdu_png_decode_u8(src_ptr, segs_ptr, n_segs, descs_ptr, n, max_row_bytes, dst_ptr, stream),
           "usdu_png_decode_u8")


PNG_GENERAL_DESC_WORDS = 16


def png_decode_general_u8(src_ptr, descs_ptr, n, max_row_bytes, dst_ptr, stream):
    """n pass descriptors (PNG_GENERAL_DESC_WORDS int64, device) over src -> u8 RGB frames in dst
    (usdu_png_decode_general_u8)."""
    _check(lib().usdu_png_decode_general_u8(src_ptr, descs_ptr, n, max_row_bytes, dst_ptr, stream),
           "usdu_png_decode_general_u8")


# baseline JPEG (include/usdu_b200.h): the host parse and Huffman decode, then the device stages
JPEG_INFO_WORDS = 16
(JI_W, JI_H, JI_COMPONENTS, JI_H0, JI_V0, JI_COLOUR, JI_RESTART, JI_MCUX, JI_MCUY, JI_BLOCKS, JI_SCAN) = range(11)
JPEG_GREY, JPEG_YCC, JPEG_RGB = 0, 1, 2
JPEG_DESC_WORDS = 16
JPEG_TILE_W = 128


def jpeg_parse(data: bytes):
    """-> (info int64 [JPEG_INFO_WORDS], quant int32 [3, 64]), or ValueError with the library's reason
    (usdu_jpeg_parse)."""
    info = np.zeros(JPEG_INFO_WORDS, np.int64)
    quant = np.zeros((3, 64), np.int32)
    st = lib().usdu_jpeg_parse(data, len(data), _i64p(info), quant.ctypes.data_as(POINTER(c_int32)))
    if st == ERR_INVALID:
        raise ValueError(lib().usdu_last_error().decode())
    _check(st, "usdu_jpeg_parse")
    return info, quant


def jpeg_decode_coefs(data: bytes, coefs: np.ndarray):
    """The Huffman decode of `data` into `coefs` (int16, 64 * info[JI_BLOCKS] words, any host memory, written in
    place), or ValueError with the library's reason (usdu_jpeg_decode_coefs)."""
    assert coefs.dtype == np.int16 and coefs.flags["C_CONTIGUOUS"]
    st = lib().usdu_jpeg_decode_coefs(data, len(data), coefs.ctypes.data, coefs.size)
    if st == ERR_INVALID:
        raise ValueError(lib().usdu_last_error().decode())
    _check(st, "usdu_jpeg_decode_coefs")


def jpeg_decode_u8(src_ptr, descs_ptr, n, n_ctas, dst_ptr, stream):
    """n frame descriptors (JPEG_DESC_WORDS int64, device) over src -> u8 RGB frames in dst (usdu_jpeg_decode_u8)."""
    _check(lib().usdu_jpeg_decode_u8(src_ptr, descs_ptr, n, n_ctas, dst_ptr, stream), "usdu_jpeg_decode_u8")


def png_encode_scratch_bytes(B: int, H: int, W: int) -> int:
    """Device scratch usdu_png_encode_u8 takes for B RGB frames [H, W, 3]."""
    raw = H * (1 + 3 * W)
    return B * ((raw + 15) // 16 * 16 + 8 * H + 16)


def png_encode_u8(src_ptr, B, H, W, C, template_ptr, png_len, runs_ptr, n_runs, chunks_ptr, n_chunks, adler_at,
                  scratch_ptr, dst_ptr, stream):
    at = (c_int64 * 4)(*[int(v) for v in adler_at])
    _check(lib().usdu_png_encode_u8(src_ptr, B, H, W, C, template_ptr, png_len, runs_ptr, n_runs, chunks_ptr, n_chunks,
                                    at, scratch_ptr, dst_ptr, stream), "usdu_png_encode_u8")


def png_decode_warps(max_row_bytes: int) -> int:
    """Ring depth (= warps per CTA) usdu_png_decode_u8 uses for rows of up to max_row_bytes on the current device."""
    r = lib().usdu_png_decode_warps(max_row_bytes)
    if r < 0:
        _check(r, "usdu_png_decode_warps")
    return r


def gather_unpack_f32(frame_ptrs_dev, n, frame_elems, dst_ptr, stream):
    """frame_ptrs_dev: device array of n u8 frame addresses; dst: device or pinned host memory (usdu_gather_unpack_f32)."""
    _check(lib().usdu_gather_unpack_f32(frame_ptrs_dev, n, frame_elems, dst_ptr, stream), "usdu_gather_unpack_f32")


# usdu_b64_png_check's table (include/usdu_b200.h)
B64_HEAD_WORDS = 24
B64_MAX_CHUNKS = 4096
B64_MAX_BLOCKS = 4096
B64_PREFIX_BYTES = 4096
B64_TABLE_WORDS = B64_HEAD_WORDS + 4 * B64_MAX_CHUNKS + 4 * B64_MAX_BLOCKS + B64_PREFIX_BYTES // 8
B64_MAX_TEXT = (1 << 31) - 17                   # the largest text it takes
(B64_CHUNKS_NONE, B64_CHUNKS_SHORT, B64_CHUNKS_PAST_END, B64_CHUNKS_AFTER_IDAT, B64_CHUNKS_IEND,
 B64_CHUNKS_FULL) = range(6)
(B64_BLOCKS_NONE, B64_BLOCKS_SHORT, B64_BLOCKS_ZLIB, B64_BLOCKS_COMPRESSED, B64_BLOCKS_LEN, B64_BLOCKS_FINAL,
 B64_BLOCKS_FULL) = range(7)


def b64_png_bytes(n: int) -> int:
    """Device bytes usdu_b64_png_check writes the decoded text of n characters to."""
    return 12 * ((n + 15) // 16)


def b64_png_check(text_ptr, n, png_ptr, table_ptr, stream):
    """text: n bytes in pinned host or device memory (16-byte aligned) -> decoded bytes at png_ptr and the verdict table
    (B64_TABLE_WORDS int64, device) at table_ptr (usdu_b64_png_check)."""
    _check(lib().usdu_b64_png_check(text_ptr, n, png_ptr, table_ptr, stream), "usdu_b64_png_check")


def t0_denoise(tiles_ptr, noise_ptr, out_ptr, n, frame, omd, stream):
    _check(lib().usdu_t0_denoise(tiles_ptr, noise_ptr, out_ptr, n, frame, omd, stream), "usdu_t0_denoise")


def mask_scratch_bytes(specs: np.ndarray) -> int:
    n = lib().usdu_mask_scratch_bytes(_i32p(specs), specs.shape[0])
    if n < 0:
        _check(int(n), "usdu_mask_scratch_bytes")
    return int(n)


def build_feather_masks(specs: np.ndarray, pool_ptr, scratch_ptr, stream):
    _check(lib().usdu_build_feather_masks(_i32p(specs), specs.shape[0], pool_ptr, scratch_ptr, stream),
           "usdu_build_feather_masks")


def tile_crop_resize(canvas_ptr, B, H, W, pitch, tiles_ptr, tabs_ptr, items_ptr, n_items, patch_w, patch_h,
                     out_ptr, flags, stream):
    _check(lib().usdu_tile_crop_resize(canvas_ptr, B, H, W, pitch, tiles_ptr, tabs_ptr, items_ptr, n_items,
                                       patch_w, patch_h, out_ptr, flags, stream), "usdu_tile_crop_resize")


def tile_blend(canvas_ptr, B, H, W, pitch, tiles_ptr, tabs_ptr, mask_ptr, items_ptr, n_items, cover_ptr, patch_w,
               patch_h, src_ptr, src_is_u8, flags, stream):
    _check(lib().usdu_tile_blend(canvas_ptr, B, H, W, pitch, tiles_ptr, tabs_ptr, mask_ptr, items_ptr, n_items,
                                 cover_ptr, patch_w, patch_h, src_ptr, int(src_is_u8), flags, stream), "usdu_tile_blend")


def plane_resample_u8(src_ptr, n, src_h, src_w, src_pitch, src_plane, tab_h_ptr, ox, ow, tab_v_ptr, oy, oh,
                      mid_y0, mid_rows, mid_ptr, dst_ptr, dst_pitch, dst_plane, stream):
    _check(lib().usdu_plane_resample_u8(src_ptr, n, src_h, src_w, src_pitch, src_plane, tab_h_ptr, ox, ow, tab_v_ptr,
                                        oy, oh, mid_y0, mid_rows, mid_ptr, dst_ptr, dst_pitch, dst_plane, stream),
           "usdu_plane_resample_u8")


def plane_pad_fill_u8(src_ptr, n, h, w, src_pitch, src_plane, hp, vp, row_index_ptr, col_index_ptr, dst_ptr,
                      dst_pitch, dst_plane, stream):
    _check(lib().usdu_plane_pad_fill_u8(src_ptr, n, h, w, src_pitch, src_plane, hp, vp, row_index_ptr, col_index_ptr,
                                        dst_ptr, dst_pitch, dst_plane, stream), "usdu_plane_pad_fill_u8")
