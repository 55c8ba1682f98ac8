"""ORACLE — test infrastructure, not product code.

ctypes binding of libskyrim_b200_probe.so (skyrim_b200/csrc/gemm_probe.cu): one launch of the wgmma GEMM per
call, with the schedule and epilogue given as raw device pointers; and of sky_probe_pangu (pangu_probe.cu): one launch
of one of Pangu's windowing kernels per call.  The product library does not export these entry points; the probe
library is the product objects plus gemm_probe.o and pangu_probe.o.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

PROBE_LIB_PATH = Path(__file__).resolve().parent.parent / "skyrim_b200" / "libskyrim_b200_probe.so"

W, W_TRI, TB, PAIR = 0, 1, 2, 3
(EPI_F32, EPI_F32_ACC, EPI_SPLIT, EPI_SPLIT_GELU, EPI_F32_STATS, EPI_GELU_STATS, EPI_REMAP, EPI_LN, EPI_LN_IMG, EPI_F16_GELU_IMG,
 EPI_F16_ROWS, EPI_GC_SILU0, EPI_GC_SILU2, EPI_GC_OUT, EPI_GC_LN0, EPI_GC_LN1, EPI_GC_LN2, EPI_QKV_WIN) = range(18)
# sky_probe_pangu (pangu_probe.cu) ops
PG_FILL_PAD, PG_ATTENTION, PG_PACK_BIAS = range(3)

_p = C.c_void_p
_i32, _i64 = C.c_int32, C.c_int64


class Geo(C.Structure):
    """mirror of sky_probe_geo_t (the engine's Geo)"""
    _fields_ = [(n, _i32) for n in ("Z", "H", "W", "C", "Hp", "nWz", "nWh", "nWw", "T", "nWin", "heads")]


class Case(C.Structure):
    """mirror of sky_probe_case_t"""
    _fields_ = [
        ("kernel", _i32), ("epi", _i32), ("block_n", _i32), ("n", _i32), ("n_valid", _i32), ("batches", _i32),
        ("grid_sms", _i32), ("nseg", _i32), ("m", _i64),
        ("a", _p * 6), ("a_bytes", _i64 * 6), ("a_batch_stride", _i64 * 6), ("a_nkb", _i32 * 6),
        ("w", _p), ("w_bytes", _i64), ("w_batch_stride", _i64), ("num_kb", _i32), ("w_rep", _i32),
        ("t", _p), ("t_bytes", _i64), ("t_batch_stride", _i64), ("t_rows", _i32), ("b_nkb_img", _i32),
        ("b_hi", _p), ("b_lo", _p), ("b_bytes", _i64), ("b_rows_per_batch", _i64), ("b_batch_bytes", _i64),
        ("out", _p), ("out_bytes", _i64), ("out_batch_stride", _i64), ("ldo", _i32), ("img_nkb", _i32),
        ("hi", _p), ("lo", _p), ("img_bytes", _i64), ("img_batch_bytes", _i64),
        ("bias", _p), ("gamma", _p), ("beta", _p), ("add", _p), ("asc", _p), ("ash", _p),
        ("csc", _p), ("csh", _p), ("t1", _p), ("vec_floats", _i64), ("add_bytes", _i64), ("t1_floats", _i64),
        ("sums", _p), ("sums_bytes", _i64), ("rows_per_batch", _i64),
        ("bdiv", _i32), ("kmul", _i32), ("kdiv", _i32), ("rb", _i32), ("same", _i32), ("eps", C.c_float),
        ("ta", _p), ("tb", _p), ("ia", _p), ("ib", _p), ("ta_bytes", _i64), ("tb_bytes", _i64), ("ta_rows", _i64),
        ("tb_rows", _i64), ("lda", _i32), ("ldb", _i32), ("yimg", _p), ("xin", _p), ("xin_img", _p), ("dstd", _p),
        ("xin_bytes", _i64), ("plane", _i64), ("nprog", _i32),
        ("geo", Geo), ("roll", _i32), ("pairs", _i32), ("part_stride", _i64),
    ]


class PanguCase(C.Structure):
    """mirror of sky_probe_pangu_t"""
    _fields_ = [
        ("op", _i32), ("geo", Geo), ("roll", _i32), ("B", _i32), ("pairs", _i32), ("n_type", _i32), ("att_nkb", _i32),
        ("part_stride", _i64), ("qkv", _p), ("qkv_bytes", _i64), ("src", _p), ("src_floats", _i64), ("tab", _p),
        ("tab_bytes", _i64), ("out", _p), ("out_bytes", _i64), ("sl2", C.c_float), ("mask_l2", C.c_float),
    ]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not PROBE_LIB_PATH.exists():
            raise RuntimeError(f"{PROBE_LIB_PATH} not found — build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(os.fspath(PROBE_LIB_PATH))
        L.sky_probe_gemm.restype = C.c_int
        L.sky_probe_gemm.argtypes = [C.POINTER(Case), C.c_void_p]
        L.sky_probe_case_size.restype = C.c_int
        L.sky_probe_case_size.argtypes = []
        L.sky_probe_pangu.restype = C.c_int
        L.sky_probe_pangu.argtypes = [C.POINTER(PanguCase), C.c_void_p]
        L.sky_probe_pangu_size.restype = C.c_int
        L.sky_probe_pangu_size.argtypes = []
        L.sky_last_error.restype = C.c_char_p
        L.sky_last_error.argtypes = []
        _lib = L
    return _lib


def make_case(**kw) -> Case:
    c = Case()
    for k, v in kw.items():
        if k in ("a", "a_bytes", "a_batch_stride", "a_nkb"):
            arr = getattr(c, k)
            for i, x in enumerate(v):
                arr[i] = x
        elif k == "geo":
            c.geo = Geo(**v)
        else:
            setattr(c, k, v)
    return c


def make_pangu_case(**kw) -> PanguCase:
    c = PanguCase()
    for k, v in kw.items():
        setattr(c, k, Geo(**v) if k == "geo" else v)
    return c


def launch(case: Case, stream: int = 0) -> tuple[int, str]:
    """(return code, error text); rc != 0 means the case was refused or the launch failed"""
    L = lib()
    rc = L.sky_probe_gemm(C.byref(case), C.c_void_p(stream))
    msg = L.sky_last_error() if rc else b""
    return rc, (msg or b"").decode()


def launch_pangu(case: PanguCase, stream: int = 0) -> tuple[int, str]:
    """sky_probe_pangu: (return code, error text)"""
    L = lib()
    rc = L.sky_probe_pangu(C.byref(case), C.c_void_p(stream))
    msg = L.sky_last_error() if rc else b""
    return rc, (msg or b"").decode()
