"""Shared by the date-function tests: the restatement of the reference's functions (tests/cpp/date_fn_oracle.c, compiled on first use into
a temporary directory), the functions in scope with their argument forms, and the calendar tables the tests run over."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from baikaldb_b200 import plan as P
from baikaldb_b200.plan import PrimitiveType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "date_fn_oracle.c")

# name -> (return type, argument types accepted besides literals, values of the extra operand: week / yearweek modes (-1 = none), extract units)
UNITS = ["year", "month", "day", "hour", "minute", "second"]
FNS = {
    "year": (T.UINT32, None), "month": (T.UINT32, None), "day": (T.UINT32, None), "dayofmonth": (T.UINT32, None), "quarter": (T.INT32, None),
    "hour": (T.UINT32, None), "minute": (T.INT32, None), "second": (T.INT32, None), "dayofweek": (T.UINT32, None), "weekday": (T.UINT32, None),
    "dayofyear": (T.UINT32, None), "week": (T.UINT32, list(range(-1, 8))), "yearweek": (T.UINT32, list(range(-1, 8))),
    "weekofyear": (T.UINT32, None), "to_days": (T.INT64, None), "to_seconds": (T.INT64, None), "unix_timestamp": (T.INT64, None),
    "datediff": (T.INT32, None), "extract": (T.UINT32, list(range(7))), "date": (T.DATE, None),
}
TIME_FNS = ("hour", "minute", "second")
OTHER_DATE = (1995 * 13 + 1) << 5 | 1          # datediff's second argument in the tests: DATE '1995-01-01'

_lib = None


def oracle():
    global _lib
    if _lib is None:
        d = os.path.join(tempfile.gettempdir(), f"bk_date_fn_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libdatefn_{int(os.path.getmtime(SRC))}.so")
        if not os.path.exists(so):
            tmp = so + f".{os.getpid()}"
            subprocess.check_call(["gcc", "-O2", "-Wall", "-Wextra", "-shared", "-fPIC", SRC, "-o", tmp])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        L.bk_oracle_date_fn.restype = ctypes.c_int64
        L.bk_oracle_date_fn.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, ctypes.c_uint64, ctypes.POINTER(ctypes.c_int)]
        L.bk_oracle_date_fn_many.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64,
                                             ctypes.c_void_p, ctypes.c_void_p]
        _lib = L
    return _lib


def oracle_one(fn, arg, prim, image, prim2=T.DATE, image2=OTHER_DATE):
    nl = ctypes.c_int(0)
    v = oracle().bk_oracle_date_fn(fn.encode(), int(arg), int(prim), int(image) & ((1 << 64) - 1), int(prim2), int(image2), ctypes.byref(nl))
    return None if nl.value else v


def expected(fn, arg, prim, images, valid=None):
    """(int64 values, validity) of fn over `images` of type `prim` (datediff: against DATE '1995-01-01'); invalid inputs give NULL"""
    x = np.ascontiguousarray(images.astype(np.uint64) if prim != T.TIME else images.astype(np.int64).view(np.uint64))
    n = len(x)
    other = np.full(n, OTHER_DATE, np.uint64)
    out, nul = np.zeros(n, np.int64), np.zeros(n, np.uint8)
    oracle().bk_oracle_date_fn_many(fn.encode(), int(arg), int(prim), x.ctypes.data, int(T.DATE), other.ctypes.data, n, out.ctypes.data, nul.ctypes.data)
    ok = nul == 0
    if valid is not None:
        ok &= valid
    return out, ok


def call(fn, x, arg=None):
    """the plan expression fn(x [, arg]) (extract: extract(unit, x); datediff: datediff(x, '1995-01-01'))"""
    if fn == "extract":
        return P.common("extract", P.str_lit(UNITS[arg] if arg < 6 else "fortnight"), x)
    if fn == "datediff":
        return P.common("datediff", x, P.str_lit("1995-01-01"))
    if fn in ("week", "yearweek") and arg is not None and arg >= 0:
        return P.common(fn, x, P.int_lit(arg))
    return P.common(fn, x)


def variants():
    """(fn, arg) pairs: every function, every mode of week / yearweek, every unit of extract and an unknown one"""
    out = []
    for fn, (_, args) in FNS.items():
        for a in (args or [0]):
            out.append((fn, a))
    return out


def date_image(y, m, d):
    return ((y * 13 + m) << 5) | d


def dt_image(y, mo, d, h=0, mi=0, s=0):
    return ((y * 13 + mo) << 46) | (d << 41) | (h << 36) | (mi << 30) | (s << 24)


def every_day():
    """DATE images of every day 0000-01-01 .. 9999-12-31, then day 0, month 0 and days 29-31 of every month of 2023 and 2024, and the zero date"""
    y = np.arange(0, 10000)
    leap = (y % 4 == 0) & ((y % 100 != 0) | (y % 400 == 0))
    lens = np.array([31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31])
    out = []
    for m in range(1, 13):
        for d in range(1, 32):
            ok = d <= lens[m - 1] + ((m == 2) & leap)
            out.append(((y[ok] * 13 + m) << 5) | d)
    days = np.sort(np.concatenate(out))
    edge = [date_image(yy, m, d) for yy in (2023, 2024) for m in range(0, 13) for d in (0, 1, 29, 30, 31)]
    return np.concatenate([days, np.array(edge + [0])]).astype(np.uint32)


def midnights():
    """TIMESTAMPs on both sides of every midnight (+08) of the uint32 range, and 0"""
    days = np.arange(0, (1 << 32) // 86400, dtype=np.int64)
    ts = np.concatenate([days * 86400 + 57599, days * 86400 + 57600, [0, (1 << 32) - 1]])
    return ts[(ts >= 0) & (ts < (1 << 32))].astype(np.uint32)


def time_sweep():
    h, mi, s = np.meshgrid(np.arange(0, 1100, 7), np.arange(0, 64, 5), np.arange(0, 64, 9), indexing="ij")
    t = ((h << 12) | (mi << 6) | s).ravel().astype(np.int32)
    return np.concatenate([t, -t]).astype(np.int32)
