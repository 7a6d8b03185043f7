"""Column batches at the boundary: Arrow layout, one values buffer + optional validity bitmap per
column, named ``"<tuple>_<slot>"`` like the reference's Arrow fields (include/expr/slot_ref.h:72-82,
src/runtime/chunk.cpp:33-92)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Tuple

import numpy as np

from .plan import PrimitiveType, storage_dtype


@dataclass
class Column:
    tuple_id: int
    slot_id: int
    prim_type: int
    values: np.ndarray                     # storage dtype (see plan.storage_dtype); (n,16) u1 for AVG blobs, (n,16400) u1 for HLL sketches,
                                           # an object array of bytes for BITMAP (rb_build_agg's serialized Roaring bitmaps)
    valid: Optional[np.ndarray] = None     # bool[n]; None = no NULLs

    @property
    def name(self) -> str:
        return f"{self.tuple_id}_{self.slot_id}"

    def __len__(self) -> int:
        return int(self.values.shape[0])

    def validity_bitmap(self) -> Optional[np.ndarray]:
        """Arrow LSB-first bitmap (1 = valid)."""
        if self.valid is None:
            return None
        return np.packbits(np.asarray(self.valid, dtype=bool), bitorder="little")

    def to_list(self) -> list:
        v = self.values
        if self.prim_type in (PrimitiveType.STRING, PrimitiveType.HLL, PrimitiveType.BITMAP):
            out = [bytes(x) for x in v]
        else:
            out = v.tolist()
        if self.valid is not None:
            out = [x if ok else None for x, ok in zip(out, self.valid.tolist())]
        return out


def make_column(tuple_id: int, slot_id: int, prim_type: int, values, valid=None) -> Column:
    if prim_type == PrimitiveType.STRING:
        arr = np.ascontiguousarray(values, dtype=np.uint8).reshape(-1, 16)
    elif prim_type == PrimitiveType.HLL:   # RAW sketches (hll_add_agg's MERGE_AGG input): 16400 bytes each
        arr = np.ascontiguousarray(values, dtype=np.uint8).reshape(-1, 16400)
    else:
        arr = np.ascontiguousarray(values, dtype=np.dtype(storage_dtype(prim_type)))
    v = None if valid is None else np.ascontiguousarray(valid, dtype=bool)
    if v is not None and v.all():
        v = None
    return Column(tuple_id, slot_id, int(prim_type), arr, v)


def unpack_validity(bitmap: Optional[np.ndarray], n: int) -> Optional[np.ndarray]:
    if bitmap is None:
        return None
    return np.unpackbits(np.asarray(bitmap, dtype=np.uint8), count=n, bitorder="little").astype(bool)


def columns_by_name(cols: Iterable[Column]) -> Dict[str, Column]:
    return {c.name: c for c in cols}


def rows_as_set(cols: List[Column], key_names: Optional[List[str]] = None) -> Dict[Tuple, Tuple]:
    """Result rows keyed by the group-key columns: the reference emits groups in hash-map iteration
    order (SURVEY.md Appendix B item 11), so results are compared as sets."""
    lists = {c.name: c.to_list() for c in cols}
    names = list(lists)
    keys = key_names if key_names is not None else names
    n = len(cols[0]) if cols else 0
    out = {}
    for i in range(n):
        k = tuple(lists[kn][i] for kn in keys)
        out[k] = tuple(lists[nm][i] for nm in names)
    return out
