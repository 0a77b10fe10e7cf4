"""ctypes driver for the UNMODIFIED reference library oracle/_ref/libduckdb_ref.so.

TEST INFRASTRUCTURE ONLY (oracle / CPU baseline): imported by tests/, by
__graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference legs.
Never imported by the product package duckdb_b200.

Uses DuckDB's public C API (src/include/duckdb.h): duckdb_open / duckdb_connect /
duckdb_query / duckdb_fetch_chunk / duckdb_vector_get_data, and the appender-free
bulk path duckdb_data_chunk + duckdb_append_data_chunk to load numpy columns.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libduckdb_ref.so")

# duckdb_type enum values (duckdb.h DUCKDB_TYPE_*)
T_BOOLEAN, T_TINYINT, T_SMALLINT, T_INTEGER, T_BIGINT = 1, 2, 3, 4, 5
T_UTINYINT, T_USMALLINT, T_UINTEGER, T_UBIGINT = 6, 7, 8, 9
T_FLOAT, T_DOUBLE = 10, 11
T_TIMESTAMP, T_DATE, T_TIME = 12, 13, 14
T_HUGEINT = 16
T_VARCHAR = 17
T_DECIMAL = 19

_NP_OF = {
    T_BOOLEAN: np.bool_, T_TINYINT: np.int8, T_SMALLINT: np.int16, T_INTEGER: np.int32,
    T_BIGINT: np.int64, T_UTINYINT: np.uint8, T_USMALLINT: np.uint16, T_UINTEGER: np.uint32,
    T_UBIGINT: np.uint64, T_FLOAT: np.float32, T_DOUBLE: np.float64, T_DATE: np.int32,
    T_TIMESTAMP: np.int64, T_TIME: np.int64,
}
_TYPE_OF_NP = {
    np.dtype(np.bool_): T_BOOLEAN, np.dtype(np.int8): T_TINYINT, np.dtype(np.int16): T_SMALLINT,
    np.dtype(np.int32): T_INTEGER, np.dtype(np.int64): T_BIGINT, np.dtype(np.uint8): T_UTINYINT,
    np.dtype(np.uint16): T_USMALLINT, np.dtype(np.uint32): T_UINTEGER, np.dtype(np.uint64): T_UBIGINT,
    np.dtype(np.float32): T_FLOAT, np.dtype(np.float64): T_DOUBLE,
}
_SQL_OF_NP = {
    np.dtype(np.bool_): "BOOLEAN", np.dtype(np.int8): "TINYINT", np.dtype(np.int16): "SMALLINT",
    np.dtype(np.int32): "INTEGER", np.dtype(np.int64): "BIGINT", np.dtype(np.uint8): "UTINYINT",
    np.dtype(np.uint16): "USMALLINT", np.dtype(np.uint32): "UINTEGER", np.dtype(np.uint64): "UBIGINT",
    np.dtype(np.float32): "FLOAT", np.dtype(np.float64): "DOUBLE",
}


def available():
    return os.path.exists(LIB_PATH)


class _Result(C.Structure):  # duckdb_result (duckdb.h): 6 deprecated words + internal_data
    _fields_ = [("a", C.c_uint64), ("b", C.c_uint64), ("c", C.c_uint64), ("d", C.c_void_p),
                ("e", C.c_void_p), ("internal_data", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("reference library not built: run python oracle/build_ref.py")
        L = C.CDLL(LIB_PATH)
        L.duckdb_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
        L.duckdb_connect.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        L.duckdb_query.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(_Result)]
        L.duckdb_result_error.argtypes = [C.POINTER(_Result)]
        L.duckdb_result_error.restype = C.c_char_p
        L.duckdb_destroy_result.argtypes = [C.POINTER(_Result)]
        L.duckdb_column_count.argtypes = [C.POINTER(_Result)]
        L.duckdb_column_count.restype = C.c_uint64
        L.duckdb_column_name.argtypes = [C.POINTER(_Result), C.c_uint64]
        L.duckdb_column_name.restype = C.c_char_p
        L.duckdb_column_type.argtypes = [C.POINTER(_Result), C.c_uint64]
        L.duckdb_column_type.restype = C.c_int
        L.duckdb_column_logical_type.argtypes = [C.POINTER(_Result), C.c_uint64]
        L.duckdb_column_logical_type.restype = C.c_void_p
        L.duckdb_decimal_internal_type.argtypes = [C.c_void_p]
        L.duckdb_decimal_internal_type.restype = C.c_int
        L.duckdb_decimal_scale.argtypes = [C.c_void_p]
        L.duckdb_decimal_scale.restype = C.c_uint8
        L.duckdb_destroy_logical_type.argtypes = [C.POINTER(C.c_void_p)]
        L.duckdb_fetch_chunk.argtypes = [_Result]
        L.duckdb_fetch_chunk.restype = C.c_void_p
        L.duckdb_data_chunk_get_size.argtypes = [C.c_void_p]
        L.duckdb_data_chunk_get_size.restype = C.c_uint64
        L.duckdb_data_chunk_get_vector.argtypes = [C.c_void_p, C.c_uint64]
        L.duckdb_data_chunk_get_vector.restype = C.c_void_p
        L.duckdb_vector_get_data.argtypes = [C.c_void_p]
        L.duckdb_vector_get_data.restype = C.c_void_p
        L.duckdb_vector_get_validity.argtypes = [C.c_void_p]
        L.duckdb_vector_get_validity.restype = C.POINTER(C.c_uint64)
        L.duckdb_destroy_data_chunk.argtypes = [C.POINTER(C.c_void_p)]
        L.duckdb_disconnect.argtypes = [C.POINTER(C.c_void_p)]
        L.duckdb_close.argtypes = [C.POINTER(C.c_void_p)]
        # appender / data chunk creation
        L.duckdb_create_logical_type.argtypes = [C.c_int]
        L.duckdb_create_logical_type.restype = C.c_void_p
        L.duckdb_create_data_chunk.argtypes = [C.POINTER(C.c_void_p), C.c_uint64]
        L.duckdb_create_data_chunk.restype = C.c_void_p
        L.duckdb_data_chunk_set_size.argtypes = [C.c_void_p, C.c_uint64]
        L.duckdb_vector_ensure_validity_writable.argtypes = [C.c_void_p]
        L.duckdb_appender_create.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]
        L.duckdb_append_data_chunk.argtypes = [C.c_void_p, C.c_void_p]
        L.duckdb_appender_error.argtypes = [C.c_void_p]
        L.duckdb_appender_error.restype = C.c_char_p
        L.duckdb_appender_destroy.argtypes = [C.POINTER(C.c_void_p)]
        L.duckdb_data_chunk_reset.argtypes = [C.c_void_p]
        L.duckdb_vector_size.restype = C.c_uint64
        _lib = L
    return _lib


class Column:
    """One result column: values (numpy), valid (bool numpy or None), scale for decimals."""

    def __init__(self, name, values, valid, type_id, scale=0):
        self.name, self.values, self.valid, self.type_id, self.scale = name, values, valid, type_id, scale


class Connection:
    def __init__(self, path=":memory:", threads=None):
        L = lib()
        self.db = C.c_void_p()
        self.con = C.c_void_p()
        if L.duckdb_open(path.encode() if path else None, C.byref(self.db)) != 0:
            raise RuntimeError("duckdb_open failed")
        if L.duckdb_connect(self.db, C.byref(self.con)) != 0:
            raise RuntimeError("duckdb_connect failed")
        if threads:
            self.execute(f"SET threads={int(threads)}")

    def close(self):
        L = lib()
        if self.con:
            L.duckdb_disconnect(C.byref(self.con))
            self.con = C.c_void_p()
        if self.db:
            L.duckdb_close(C.byref(self.db))
            self.db = C.c_void_p()

    def execute(self, sql):
        """Run sql; return list[Column] (numeric columns as numpy; VARCHAR as list of str/None)."""
        L = lib()
        res = _Result()
        state = L.duckdb_query(self.con, sql.encode(), C.byref(res))
        if state != 0:
            msg = L.duckdb_result_error(C.byref(res))
            msg = msg.decode() if msg else "unknown error"
            L.duckdb_destroy_result(C.byref(res))
            raise RuntimeError(msg)
        ncols = L.duckdb_column_count(C.byref(res))
        names, types, scales, phys = [], [], [], []
        for i in range(ncols):
            names.append(L.duckdb_column_name(C.byref(res), i).decode())
            t = L.duckdb_column_type(C.byref(res), i)
            types.append(t)
            sc, ph = 0, t
            if t == T_DECIMAL:
                lt = C.c_void_p(L.duckdb_column_logical_type(C.byref(res), i))
                ph = L.duckdb_decimal_internal_type(lt)
                sc = L.duckdb_decimal_scale(lt)
                L.duckdb_destroy_logical_type(C.byref(lt))
            scales.append(sc)
            phys.append(ph)
        parts = [[] for _ in range(ncols)]
        valids = [[] for _ in range(ncols)]
        while True:
            chunk = L.duckdb_fetch_chunk(res)
            if not chunk:
                break
            chunk = C.c_void_p(chunk)
            n = L.duckdb_data_chunk_get_size(chunk)
            for i in range(ncols):
                vec = L.duckdb_data_chunk_get_vector(chunk, i)
                data = L.duckdb_vector_get_data(vec)
                val = L.duckdb_vector_get_validity(vec)
                if val:
                    words = np.ctypeslib.as_array(val, shape=((n + 63) // 64,)).copy()
                    bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)
                else:
                    bits = np.ones(n, dtype=bool)
                valids[i].append(bits)
                ph = phys[i]
                if ph in _NP_OF:
                    dt = np.dtype(_NP_OF[ph])
                    buf = (C.c_char * (n * dt.itemsize)).from_address(data) if n else b""
                    parts[i].append(np.frombuffer(buf, dtype=dt, count=n).copy())
                elif ph == T_HUGEINT:
                    buf = (C.c_char * (n * 16)).from_address(data) if n else b""
                    raw = np.frombuffer(buf, dtype=np.uint64, count=2 * n).copy().reshape(n, 2)
                    # python ints: upper is signed
                    vals = raw[:, 1].astype(np.int64).astype(object) * (1 << 64) + raw[:, 0].astype(object)
                    parts[i].append(vals)
                elif ph == T_VARCHAR:
                    # string_t: 4-byte length, then up to 12 inlined bytes or a 4-byte prefix and a pointer
                    raw = np.frombuffer((C.c_char * (n * 16)).from_address(data), dtype=np.uint8).reshape(n, 16) \
                        if n else np.zeros((0, 16), np.uint8)
                    lens = raw[:, :4].copy().view(np.uint32)[:, 0]
                    inlined = np.frombuffer(raw[:, 4:].tobytes(), dtype="S12")  # trailing NUL bytes dropped
                    # all at once where the bytes after the string are zero, so the S12 value is the string
                    fast = bits & (lens <= 12) & (np.char.str_len(inlined) == lens)
                    out = np.empty(n, dtype=object)
                    out[fast] = [s.decode("utf8", "replace") for s in inlined[fast].tolist()]
                    for r in np.flatnonzero(bits & ~fast):
                        base = data + int(r) * 16
                        ln = int(lens[r])
                        if ln <= 12:
                            out[r] = C.string_at(base + 4, ln).decode("utf8", "replace")
                        else:
                            ptr = C.c_void_p.from_address(base + 8).value
                            out[r] = C.string_at(ptr, ln).decode("utf8", "replace")
                    parts[i].append(out)
                else:
                    raise RuntimeError(f"unsupported result type {ph} for column {names[i]}")
            L.duckdb_destroy_data_chunk(C.byref(chunk))
        L.duckdb_destroy_result(C.byref(res))
        cols = []
        for i in range(ncols):
            if parts[i]:
                vals = np.concatenate(parts[i])
                valid = np.concatenate(valids[i])
            else:
                vals = np.zeros(0, dtype=_NP_OF.get(phys[i], object))
                valid = np.zeros(0, dtype=bool)
            cols.append(Column(names[i], vals, None if valid.all() else valid, types[i], scales[i]))
        return cols

    def fetchall(self, sql):
        """Rows as python tuples (None for NULL); decimals as scaled ints."""
        cols = self.execute(sql)
        n = len(cols[0].values) if cols else 0
        rows = []
        for r in range(n):
            row = []
            for c in cols:
                if c.valid is not None and not c.valid[r]:
                    row.append(None)
                else:
                    v = c.values[r]
                    row.append(v.item() if hasattr(v, "item") else v)
            rows.append(tuple(row))
        return rows

    def load_table(self, name, columns):
        """CREATE TABLE name and bulk-append numpy columns.
        columns: dict name -> ndarray | (ndarray, valid_bool_ndarray)."""
        L = lib()
        defs, arrays, valids = [], [], []
        for cname, col in columns.items():
            valid = None
            if isinstance(col, tuple):
                col, valid = col
            col = np.ascontiguousarray(col)
            defs.append(f"{cname} {_SQL_OF_NP[col.dtype]}")
            arrays.append(col)
            valids.append(valid)
        self.execute(f"CREATE TABLE {name} ({', '.join(defs)})")
        n = len(arrays[0]) if arrays else 0
        app = C.c_void_p()
        if L.duckdb_appender_create(self.con, None, name.encode(), C.byref(app)) != 0:
            raise RuntimeError("appender_create failed")
        ltypes = (C.c_void_p * len(arrays))(*[L.duckdb_create_logical_type(_TYPE_OF_NP[a.dtype]) for a in arrays])
        chunk = C.c_void_p(L.duckdb_create_data_chunk(ltypes, len(arrays)))
        vsize = L.duckdb_vector_size()
        for start in range(0, n, vsize):
            cnt = min(vsize, n - start)
            L.duckdb_data_chunk_reset(chunk)
            for i, a in enumerate(arrays):
                vec = L.duckdb_data_chunk_get_vector(chunk, i)
                dst = L.duckdb_vector_get_data(vec)
                C.memmove(dst, a.ctypes.data + start * a.itemsize, cnt * a.itemsize)
                if valids[i] is not None:
                    L.duckdb_vector_ensure_validity_writable(vec)
                    vptr = L.duckdb_vector_get_validity(vec)
                    bits = np.zeros(((cnt + 63) // 64) * 64, dtype=np.uint8)
                    bits[:cnt] = valids[i][start:start + cnt]
                    words = np.packbits(bits, bitorder="little").view(np.uint64)
                    C.memmove(vptr, words.ctypes.data, words.nbytes)
            L.duckdb_data_chunk_set_size(chunk, cnt)
            if L.duckdb_append_data_chunk(app, chunk) != 0:
                raise RuntimeError("append_data_chunk failed: %s" % L.duckdb_appender_error(app))
        L.duckdb_destroy_data_chunk(C.byref(chunk))
        for i in range(len(arrays)):
            lt = C.c_void_p(ltypes[i])
            L.duckdb_destroy_logical_type(C.byref(lt))
        L.duckdb_appender_destroy(C.byref(app))
