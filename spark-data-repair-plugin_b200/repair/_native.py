"""ctypes binding of ``libb200repair.so`` (C ABI declared in ``include/b200repair.h``).

This is the only door into the hand-written sm_90a kernels.  There is no CPU fallback: if the
shared library is missing, or no CUDA device is usable, every engine entry point raises.

Adding an entry point: declare it in the header, give it a row in ``_SIGNATURES`` (the argument
kinds below do the marshalling), and add a ``Context`` method -- one ``_call`` when the Python
arguments map one-to-one onto the C ones.  Every public ``Context`` method outside ``_NOT_PROFILED`` is
profiled.
"""
import ctypes
import functools
import os
from ctypes import POINTER, byref, c_char_p, c_double, c_int, c_int32, c_int64, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_NAME = "libb200repair.so"
LIB_PATH = os.path.join(_HERE, LIB_NAME)

DR_OP = {"EQ": 0, "IQ": 1, "LT": 2, "GT": 3}


class NativeError(RuntimeError):
    pass


class dr_forest(ctypes.Structure):
    _fields_ = [
        ("n_seq", c_int32), ("n_trees", c_int32), ("n_nodes", c_int32), ("n_feat", c_int32),
        ("seq_tree_off", c_void_p), ("tree_node_off", c_void_p), ("node_thr", c_void_p),
        ("node_meta", c_void_p), ("baseline", c_void_p), ("feat_col", c_void_p),
        ("enc_lut_off", c_void_p), ("enc_lut", c_void_p), ("class_code", c_void_p),
        ("kind", c_int32), ("integral", c_int32), ("n_classes", c_int32),
    ]


class dr_forest_ranked(ctypes.Structure):
    _fields_ = [
        ("n_seq", c_int32), ("n_trees", c_int32), ("n_nodes", c_int32), ("n_leaves", c_int32),
        ("n_slots", c_int32), ("max_depth", c_int32), ("n_chunks", c_int32), ("layout", c_int32),
        ("chunk_tree_off", c_void_p), ("chunk_seq", c_void_p), ("chunk_node_off", c_void_p),
        ("chunk_leaf_off", c_void_p), ("chunk_hdr_off", c_void_p), ("tree_hdr", c_void_p),
        ("node_word", c_void_p), ("leaf_value", c_void_p), ("baseline", c_void_p), ("slot_col", c_void_p),
        ("rank_lut_off", c_void_p), ("rank_lut", c_void_p), ("slot_nan", c_void_p), ("class_code", c_void_p),
        ("n_classes", c_int32),
    ]


class dr_domain_target(ctypes.Structure):
    _fields_ = [("target", c_void_p), ("bitmap", c_void_p), ("hist_t", c_void_p), ("dom_t", c_int32),
                ("n_corr", c_int32), ("corr", c_void_p * 8), ("cooc", c_void_p * 8), ("tau", c_int64 * 8),
                ("dom_c", c_int32 * 8)]


class dr_gbdt_params(ctypes.Structure):
    _fields_ = [("n_rows", c_int32), ("n_features", c_int32), ("n_classes", c_int32), ("n_iter", c_int32),
                ("max_depth", c_int32), ("num_leaves", c_int32), ("min_data_in_leaf", c_int32),
                ("learning_rate", c_double), ("min_sum_hessian", c_double), ("qscale", c_double),
                ("reg_lambda", c_double), ("colsample_bytree", c_double), ("subsample", c_double),
                ("subsample_freq", c_int32), ("seed", c_int32)]


class dr_gbdt_boost(ctypes.Structure):
    _fields_ = [("boosting", c_int32), ("goss_warmup", c_int32), ("goss_top_k", c_int32), ("goss_other_k", c_int32),
                ("reg_alpha", c_double), ("min_split_gain", c_double), ("drop_off", c_void_p), ("drop_iter", c_void_p)]


DR_GBDT_BOOST = {"gbdt": 0, "dart": 1, "goss": 2, "rf": 3}


class dr_hll_pair(ctypes.Structure):
    _fields_ = [("hx", c_void_p), ("y_data", c_void_p), ("y_off", c_void_p), ("bits", c_void_p), ("regs", c_void_p),
                ("dom_x", c_int32), ("dom_y", c_int32), ("y_kind", c_int32)]


# value kinds of dr_hll_dict / dr_hll_pairs by Spark type (byte / short / boolean travel as int32)
DR_HLL_KIND = {"string": 0, "int": 1, "boolean": 1, "long": 2, "float": 3, "double": 4}


# ---- argument kinds --------------------------------------------------------------------------------
# Pointer-width ctypes types whose from_param converts a Python value at call time.  ctypes keeps what
# from_param returns alive until the C function returns, so the host arrays built here need no other
# reference.
def _address(buf):
    return buf if buf is None or isinstance(buf, int) else buf.data_ptr()


class _Buf(c_void_p):
    """A buffer: a torch tensor (its data_ptr()), an integer address, or None for NULL."""

    @classmethod
    def from_param(cls, buf):
        return c_void_p(_address(buf))


class _Bufs(c_void_p):
    """A list of buffers, each as _Buf takes it, passed as a host void* array."""

    @classmethod
    def from_param(cls, bufs):
        return (c_void_p * max(len(bufs), 1))(*[_address(b) for b in bufs])


class _Ints(c_void_p):
    """A list of integers passed as a host array of _elem, or None for NULL."""
    _elem = None

    @classmethod
    def from_param(cls, vals):
        return None if vals is None else (cls._elem * max(len(vals), 1))(*[int(v) for v in vals])


class _I32s(_Ints):
    _elem = c_int32


class _I64s(_Ints):
    _elem = c_int64


_SIGNATURES = {
    # name: (restype, argtypes)
    "dr_ctx_create": (c_int, [c_int, POINTER(c_void_p)]),
    "dr_ctx_destroy": (c_int, [c_void_p]),
    "dr_last_error": (c_char_p, [c_void_p]),
    "dr_abi_version": (c_int, []),
    "dr_launch_count": (c_int64, [c_void_p]),
    "dr_widen_u8": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_void_p]),
    "dr_h2d_copy": (c_int, [c_void_p, _Bufs, _Bufs, _I64s, c_int, c_int, c_void_p]),
    "dr_d2h_copy": (c_int, [c_void_p, _Bufs, _Bufs, _I64s, c_int, c_int, c_void_p]),
    "dr_index_presence": (c_int, [c_void_p, _Buf, c_int, _Buf, c_int64, c_int64, c_int32, _Buf, c_void_p]),
    "dr_index_remap": (c_int, [c_void_p, _Buf, c_int, _Buf, c_int64, c_int64, _Buf, c_int32, _Buf, c_void_p]),
    "dr_ids_unique_i64": (c_int, [c_void_p, _Buf, c_int64, POINTER(c_int), c_void_p]),
    "dr_gather_i64": (c_int, [c_void_p, _Buf, _Buf, c_int64, _Buf, c_void_p]),
    "dr_valid_bits": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_void_p]),
    "dr_scan_hist": (c_int, [c_void_p, _Bufs, _I32s, c_int, c_int64, _Bufs, _Buf, c_void_p]),
    "dr_lut_scan": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int32, _Buf, c_void_p]),
    "dr_quartiles": (c_int, [c_void_p, _Buf, c_int64, POINTER(c_double), POINTER(c_int64), c_void_p]),
    "dr_range_flag": (c_int, [c_void_p, _Buf, c_int64, c_double, c_double, _Buf, c_void_p]),
    "dr_lof_score": (c_int, [c_void_p, _Buf, _Buf, c_int64, c_int32, _Buf, _Buf, _Buf, _Buf, c_void_p]),
    "dr_lof_median": (c_int, [c_void_p, _Buf, c_int64, c_int64, c_int64, POINTER(c_int64), c_void_p]),
    "dr_lof_flag": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int32, c_int32, _Buf, c_void_p]),
    "dr_dc_const": (c_int, [c_void_p, _Bufs, _I32s, _I32s, c_int, c_int64, _Buf, c_void_p]),
    "dr_dc_fd_build": (c_int, [c_void_p, _Bufs, _I64s, c_int, _Buf, c_int64, c_int64, _Buf, _Buf, c_void_p]),
    "dr_dc_fd_flag": (c_int, [c_void_p, _Bufs, _I64s, c_int, c_int64, c_int64, _Buf, _Buf, _Buf, c_void_p]),
    "dr_dc_hash_build": (c_int, [c_void_p, _Bufs, _I64s, c_int, _Buf, c_int64, c_int64, _Buf, _Buf, _Buf,
                                 c_void_p]),
    "dr_dc_hash_flag": (c_int, [c_void_p, _Bufs, _I64s, c_int, _Buf, c_int, c_int64, c_int64, _Buf, _Buf, _Buf,
                                _Buf, c_void_p]),
    "dr_dc_lt_flag": (c_int, [c_void_p, _Bufs, _I64s, c_int, _Buf, c_int64, c_int64, _Buf, _Buf, c_void_p]),
    "dr_bitmap_or": (c_int, [c_void_p, _Buf, _Buf, c_int64, c_void_p]),
    "dr_bitmap_andnot": (c_int, [c_void_p, _Buf, _Buf, c_int64, c_void_p]),
    "dr_bitmap_count": (c_int, [c_void_p, _Buf, c_int64, POINTER(c_int64), c_void_p]),
    "dr_bitmap_count_many": (c_int, [c_void_p, _Bufs, c_int, c_int64, POINTER(c_int64), c_void_p]),
    "dr_bitmap_to_rows_async": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int64, c_void_p]),
    "dr_bitmaps_to_rows_many": (c_int, [c_void_p, _Bufs, c_int, c_int64, _Bufs, _I64s, c_void_p]),
    "dr_bitmap_to_rows": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int64, POINTER(c_int64), c_void_p]),
    "dr_bitmap_rows_after_count": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int64, c_void_p]),
    "dr_tile_null_bitmaps": (c_int, [c_void_p, _Buf, c_int64, c_int, c_int64, _Buf, c_void_p]),
    "dr_changed_bitmap": (c_int, [c_void_p, _Buf, _Buf, c_int64, _Buf, c_void_p]),
    "dr_bitmap_gather": (c_int, [c_void_p, _Buf, _Buf, c_int64, _Buf, c_void_p]),
    "dr_bitmap_clear_rows": (c_int, [c_void_p, _Buf, _Buf, _Buf, c_int64, c_void_p]),
    "dr_discretize": (c_int, [c_void_p, _Buf, c_int64, c_double, c_double, c_int32, _Buf, c_void_p]),
    "dr_pair_presence": (c_int, [c_void_p, _Bufs, _I32s, c_int, _I32s, _I32s, c_int, _I64s, c_int64, c_int64,
                                 c_int64, _Buf, c_void_p]),
    "dr_cooc": (c_int, [c_void_p, _Bufs, _I32s, c_int, _I32s, _I32s, c_int, _I64s, c_int64, _Buf, c_void_p]),
    "dr_domain_score": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int32, _Bufs, _I32s, _Bufs, c_int, _Buf, _I64s,
                                c_int64, c_double, _Buf, _Buf, _Buf, c_void_p]),
    "dr_domain_prune": (c_int, [c_void_p, POINTER(dr_domain_target), c_int, c_int64, c_int64, c_double, _Buf,
                                c_void_p]),
    "dr_gather_rows_masked": (c_int, [c_void_p, _Bufs, _Bufs, c_int, _Buf, c_int64, _Buf, c_void_p]),
    "dr_gather_rows_masked_f64": (c_int, [c_void_p, _Bufs, _Bufs, c_int, _Buf, c_int64, _Buf, c_void_p]),
    "dr_gather_rows_masked_nulls": (c_int, [c_void_p, _Bufs, _Bufs, c_int, _Buf, c_int64, _Buf, _Buf, c_int64,
                                            c_void_p]),
    "dr_tile_null_bitmap": (c_int, [c_void_p, _Buf, c_int64, c_int, c_int, _Buf, c_void_p]),
    "dr_tile_null_bitmap_f64": (c_int, [c_void_p, _Buf, c_int64, c_int, c_int, _Buf, c_void_p]),
    "dr_gather_i32": (c_int, [c_void_p, _Buf, _Buf, c_int64, _Buf, c_void_p]),
    "dr_gather_f64": (c_int, [c_void_p, _Buf, _Buf, c_int64, _Buf, c_void_p]),
    "dr_tile_gather_i32": (c_int, [c_void_p, _Buf, c_int, c_int, _Buf, c_int64, _Buf, c_void_p]),
    "dr_tile_gather_f64": (c_int, [c_void_p, _Buf, c_int, c_int, _Buf, c_int64, _Buf, c_void_p]),
    "dr_lookup_sorted": (c_int, [c_void_p, _Buf, c_int64, _Buf, c_int64, _Buf, c_void_p]),
    "dr_forest_predict": (c_int, [c_void_p, POINTER(dr_forest), _Buf, c_int, _Buf, c_int, _Buf, c_int64, c_int,
                                  _Buf, c_void_p]),
    "dr_cooc_skip": (c_int, [c_void_p, _Bufs, _I32s, c_int, _I32s, _I32s, c_int, _I64s, c_int64, _Buf, _I64s,
                             _Buf, c_void_p]),
    "dr_key_presence": (c_int, [c_void_p, _Bufs, _I64s, c_int, c_int64, c_int64, _Buf, c_void_p]),
    "dr_key_flag": (c_int, [c_void_p, _Bufs, _I64s, c_int, c_int64, c_int64, _Buf, _Buf, c_void_p]),
    "dr_dc_exists": (c_int, [c_void_p, _Bufs, _Bufs, _I32s, c_int, c_int64, _Buf, _Buf, _Buf, c_void_p]),
    "dr_combine_counts": (c_int, [c_void_p, _Buf, c_int, c_int64, _I64s, _I32s, c_int, _Buf, c_void_p]),
    "dr_forest_predict_ranked": (c_int, [c_void_p, POINTER(dr_forest_ranked), _Buf, c_int, _Buf, c_int64, c_int,
                                         _Buf, c_void_p]),
    "dr_gbdt_workspace_bytes": (c_int64, [c_int32, c_int32]),
    "dr_gbdt_train": (c_int, [c_void_p, POINTER(dr_gbdt_params), _Buf, _I32s, _Buf, _Buf, _Buf, POINTER(c_double),
                              _Buf, c_int64, _Buf, _Buf, c_void_p]),
    "dr_gbdt_train_ex_workspace_bytes": (c_int64, [c_int32, c_int32, c_int64]),
    "dr_gbdt_train_ex": (c_int, [c_void_p, POINTER(dr_gbdt_params), POINTER(dr_gbdt_boost), _Buf, _I32s, _Buf, _Buf,
                                 _Buf, POINTER(c_double), _Buf, c_int64, _Buf, _Buf, c_void_p]),
    "dr_tile_fill_i32": (c_int, [c_void_p, _Buf, c_int, c_int, _Buf, c_int64, c_int32, c_void_p]),
    "dr_scatter_i32": (c_int, [c_void_p, _Buf, _Buf, _Buf, c_int64, c_void_p]),
    "dr_scatter_f64": (c_int, [c_void_p, _Buf, _Buf, _Buf, c_int64, c_void_p]),
    "dr_fd_map_build": (c_int, [c_void_p, _Buf, _Buf, _Buf, _Buf, c_int64, c_int32, _Buf, _Buf, c_void_p]),
    "dr_tile_lut_fill": (c_int, [c_void_p, _Buf, c_int, c_int, c_int, _Buf, c_int64, _Buf, c_int32, c_void_p]),
    "dr_kmeans_assign": (c_int, [c_void_p, _Bufs, _I32s, _I64s, c_int, c_int64, _Buf, c_int64, _Buf, c_int32, _Buf,
                                 c_int32, _Buf, c_void_p]),
    "dr_label_counts": (c_int, [c_void_p, _Buf, _Buf, c_int32, c_int64, c_int32, c_int32, _Buf, c_void_p]),
    "dr_error_map": (c_int, [c_void_p, _Bufs, c_int, c_int64, _Buf, c_void_p]),
    "dr_null_bits": (c_int, [c_void_p, _Buf, c_int64, c_int64, c_int64, c_uint64, c_double, _Buf, c_void_p]),
    "dr_flatten": (c_int, [c_void_p, _Bufs, _I64s, c_int, c_int64, _Buf, _Buf, _Buf, _Buf, c_void_p]),
    "dr_hll_dict": (c_int, [c_void_p, c_int32, _Buf, _Buf, c_int64, _Buf, _Buf, c_void_p]),
    "dr_hll_pairs": (c_int, [c_void_p, POINTER(dr_hll_pair), c_int, c_void_p]),
}

EXPORTED_SYMBOLS = tuple(sorted(_SIGNATURES))

_lib = None


def load_library():
    """dlopen the in-tree shared library and bind every entry point; raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeError(
            "{} not found next to {} -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)".format(LIB_NAME, __file__))
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


class Context:
    """One ``dr_ctx`` (one GPU).  Methods take torch CUDA tensors purely as device-buffer carriers."""

    def __init__(self, device_index):
        import torch
        self.profile = None  # set to [] to collect (name, start_event, end_event) per C-ABI call
        if not torch.cuda.is_available():
            raise NativeError("no CUDA device is available; the repair engine has no CPU fallback")
        self.lib = load_library()
        self.device_index = int(device_index)
        self._h = c_void_p()
        rc = self.lib.dr_ctx_create(self.device_index, byref(self._h))
        if rc != 0:
            msg = self.lib.dr_last_error(self._h).decode() if self._h else "dr_ctx_create failed"
            raise NativeError(msg)

    def close(self):
        if getattr(self, "_h", None):
            self.lib.dr_ctx_destroy(self._h)
            self._h = None

    # One pooled context per device for the public API: a RepairModel.run() borrows it instead of creating
    # (cudaMallocHost + cudaMalloc) and destroying (cudaFree: a device synchronisation) its own, and the scratch
    # buffer it has grown stays grown for the next run.  A dr_ctx is not thread-safe: one run at a time per device.
    _pool = {}

    @classmethod
    def acquire(cls, device_index):
        ctx = cls._pool.pop(int(device_index), None)
        if ctx is None or not getattr(ctx, "_h", None):
            ctx = cls(device_index)
        ctx.profile = None
        ctx.launches_at_acquire = ctx.launch_count
        return ctx

    @classmethod
    def release(cls, ctx):
        if ctx is None or not getattr(ctx, "_h", None):
            return
        if int(ctx.device_index) in cls._pool:
            ctx.close()
        else:
            cls._pool[int(ctx.device_index)] = ctx

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _call(self, name, *args):
        """lib.<name>(context, *args, current torch stream); raises NativeError on a non-zero return code."""
        import torch
        if getattr(self.lib, name)(self._h, *args, torch.cuda.current_stream().cuda_stream) != 0:
            raise NativeError("libb200repair: " + self.lib.dr_last_error(self._h).decode())

    @property
    def launch_count(self):
        return int(self.lib.dr_launch_count(self._h))

    def widen_u8(self, src, n, dst):
        self._call("dr_widen_u8", src, n, dst)

    # ---- Arrow ingest / egress ---------------------------------------------------------------------
    def h2d_copy(self, host_ptrs, dev_tensors_or_ptrs, nbytes, threads=0):
        """Pageable host buffers (addresses) -> device (tensors or addresses); blocks until complete."""
        self._call("dr_h2d_copy", host_ptrs, dev_tensors_or_ptrs, nbytes, len(host_ptrs), threads)

    def d2h_copy(self, dev_tensors_or_ptrs, host_ptrs, nbytes, threads=0):
        self._call("dr_d2h_copy", dev_tensors_or_ptrs, host_ptrs, nbytes, len(host_ptrs), threads)

    def index_presence(self, idx_ptr, width, validity_ptr, bit_offset, n_rows, dict_size, used):
        self._call("dr_index_presence", idx_ptr, width, validity_ptr, bit_offset, n_rows, dict_size, used)

    def index_remap(self, idx_ptr, width, validity_ptr, bit_offset, n_rows, lut_ptr, dict_size, dst_ptr):
        self._call("dr_index_remap", idx_ptr, width, validity_ptr, bit_offset, n_rows, lut_ptr, dict_size, dst_ptr)

    def ids_unique(self, ids, n):
        out = c_int()
        self._call("dr_ids_unique_i64", ids, n, byref(out))
        return bool(out.value)

    def gather_i64(self, col, rows, n, out):
        self._call("dr_gather_i64", col, rows, n, out)

    def valid_bits(self, codes, n, bits):
        self._call("dr_valid_bits", codes, n, bits)

    # ---- detectors -------------------------------------------------------------------------------
    def scan_hist(self, cols, dom, n_rows, bitmaps, hist):
        self._call("dr_scan_hist", cols, dom, len(cols), n_rows, bitmaps, hist)

    def lut_scan(self, col, n_rows, lut, dict_size, bitmap):
        self._call("dr_lut_scan", col, n_rows, lut, dict_size, bitmap)

    def quartiles(self, col, n_rows):
        q = (c_double * 2)()
        n = c_int64()
        self._call("dr_quartiles", col, n_rows, q, byref(n))
        return float(q[0]), float(q[1]), int(n.value)

    def range_flag(self, col, n_rows, lower, upper, bitmap):
        self._call("dr_range_flag", col, n_rows, lower, upper, bitmap)

    def lof_score(self, u, cnt, k, verdict, kdist, lrd, lof=None):
        """LOF over sorted distinct values u (float64) with multiplicities cnt (int64), all device tensors of
        one length; writes verdict (uint8, 1 = outlier), kdist and lrd, and lof when given."""
        self._call("dr_lof_score", u, cnt, int(u.numel()), int(k), verdict, kdist, lrd, lof)

    def lof_median(self, cnt, r0, r1):
        """-> (entry holding rank r0, entry holding rank r1) of the multiset counted by cnt (device int64)."""
        out = (c_int64 * 2)()
        self._call("dr_lof_median", cnt, int(cnt.numel()), int(r0), int(r1), out)
        return int(out[0]), int(out[1])

    def lof_flag(self, col, n_rows, verdict, dict_size, null_verdict, bitmap):
        self._call("dr_lof_flag", col, n_rows, verdict, dict_size, int(bool(null_verdict)), bitmap)

    def dc_const(self, cols, ops, args, n_rows, row_bitmap):
        self._call("dr_dc_const", cols, ops, args, len(cols), n_rows, row_bitmap)

    def dc_fd_build(self, key_cols, strides, b_col, n_rows, key_space, lo, hi):
        self._call("dr_dc_fd_build", key_cols, strides, len(key_cols), b_col, n_rows, key_space, lo, hi)

    def dc_fd_flag(self, key_cols, strides, n_rows, key_space, lo, hi, row_bitmap):
        self._call("dr_dc_fd_flag", key_cols, strides, len(key_cols), n_rows, key_space, lo, hi, row_bitmap)

    def dc_hash_build(self, key_cols, strides, b_col, n_rows, capacity, table_keys, lo, hi):
        self._call("dr_dc_hash_build", key_cols, strides, len(key_cols), b_col, n_rows, capacity, table_keys, lo, hi)

    def dc_hash_flag(self, key_cols, strides, x_col, mode, n_rows, capacity, table_keys, lo, hi, row_bitmap):
        self._call("dr_dc_hash_flag", key_cols, strides, len(key_cols), x_col, mode, n_rows, capacity, table_keys,
                   lo, hi, row_bitmap)

    def dc_lt_flag(self, key_cols, strides, x_col, n_rows, key_space, hi, row_bitmap):
        self._call("dr_dc_lt_flag", key_cols, strides, len(key_cols), x_col, n_rows, key_space, hi, row_bitmap)

    # ---- bitmaps ---------------------------------------------------------------------------------
    def bitmap_or(self, dst, src, n_rows):
        self._call("dr_bitmap_or", dst, src, n_rows)

    def bitmap_andnot(self, dst, src, n_rows):
        self._call("dr_bitmap_andnot", dst, src, n_rows)

    def bitmap_count(self, bitmap, n_rows):
        n = c_int64()
        self._call("dr_bitmap_count", bitmap, n_rows, byref(n))
        return int(n.value)

    def bitmap_count_many(self, bitmaps, n_rows):
        """Popcounts of several bitmaps with one host synchronisation."""
        out = []
        for i in range(0, len(bitmaps), 128):
            part = bitmaps[i:i + 128]
            counts = (c_int64 * len(part))()
            self._call("dr_bitmap_count_many", part, len(part), n_rows, counts)
            out += [int(c) for c in counts]
        return out

    def bitmap_to_rows_async(self, bitmap, n_rows, out_rows, count):
        """Ordered compaction of a bitmap whose popcount is known: no host synchronisation."""
        self._call("dr_bitmap_to_rows_async", bitmap, n_rows, out_rows, count)

    def bitmaps_to_rows_many(self, bitmaps, n_rows, outs, counts):
        """Ordered compaction of several bitmaps with known popcounts (three launches per 128 bitmaps)."""
        for i in range(0, len(bitmaps), 128):
            part, part_counts = bitmaps[i:i + 128], counts[i:i + 128]
            part_outs = [o if c else None for o, c in zip(outs[i:i + 128], part_counts)]
            self._call("dr_bitmaps_to_rows_many", part, len(part), n_rows, part_outs, part_counts)

    def bitmap_to_rows(self, bitmap, n_rows, out_rows, capacity):
        n = c_int64()
        self._call("dr_bitmap_to_rows", bitmap, n_rows, out_rows, capacity, byref(n))
        return int(n.value)

    def bitmap_rows_after_count(self, bitmap, n_rows, out_rows, capacity):
        self._call("dr_bitmap_rows_after_count", bitmap, n_rows, out_rows, capacity)

    def tile_null_bitmaps(self, tile, n, n_cols, words_per_col, out):
        self._call("dr_tile_null_bitmaps", tile, n, n_cols, words_per_col, out)

    def changed_bitmap(self, current, repaired, n, out):
        self._call("dr_changed_bitmap", current, repaired, n, out)

    def bitmap_gather(self, src, rows, n, out):
        self._call("dr_bitmap_gather", src, rows, n, out)

    def bitmap_clear_rows(self, bitmap, rows, flags, n):
        self._call("dr_bitmap_clear_rows", bitmap, rows, flags, n)

    # ---- statistics ------------------------------------------------------------------------------
    def discretize(self, vals, n_rows, vmin, denom, thres, out):
        self._call("dr_discretize", vals, n_rows, vmin, denom, thres, out)

    def pair_presence(self, cols, dom, px, py, bit_off, n_rows, block_rows, n_blocks, bits):
        self._call("dr_pair_presence", cols, dom, len(cols), px, py, len(px), bit_off, n_rows, block_rows, n_blocks,
                   bits)

    def cooc(self, cols, dom, px, py, tab_off, n_rows, out):
        self._call("dr_cooc", cols, dom, len(cols), px, py, len(px), tab_off, n_rows, out)

    def cooc_skip(self, cols, dom, px, py, tab_off, n_rows, skip, skip_off, out):
        """dr_cooc with one uncounted entry per x value (skip: device int32 or None)."""
        self._call("dr_cooc_skip", cols, dom, len(cols), px, py, len(px), tab_off, n_rows, skip,
                   skip_off if skip is not None else None, out)

    def key_presence(self, cols, strides, n_rows, space, bits):
        self._call("dr_key_presence", cols, strides, len(cols), n_rows, space, bits)

    def key_flag(self, cols, strides, n_rows, space, viol_bits, row_bitmap):
        self._call("dr_key_flag", cols, strides, len(cols), n_rows, space, viol_bits, row_bitmap)

    def dc_exists(self, left, right, signs, n, group_begin, group_end, out):
        self._call("dr_dc_exists", left, right, signs, len(signs), n, group_begin, group_end, out)

    def combine_counts(self, gathered, world, n, seg_off, seg_op, out):
        self._call("dr_combine_counts", gathered, world, n, seg_off, seg_op, len(seg_op), out)

    def domain_score(self, rows, n_cells, target, dom_t, corr, dom_c, cooc, hist_t, tau, n_total, beta, out_top1,
                     out_prob, out_weak):
        self._call("dr_domain_score", rows, n_cells, target, dom_t, corr, dom_c, cooc, len(corr), hist_t, tau,
                   n_total, beta, out_top1, out_prob, out_weak)

    def domain_prune(self, targets, n_rows, n_total, beta, removed):
        """targets: [(target col, bitmap, hist_t ptr, dom_t, [(corr col, cooc ptr, dom_c, tau)])] -- pointers
        are device addresses (ints) or tensors; removed: device int64[len(targets)], accumulated."""
        arr = (dr_domain_target * max(len(targets), 1))()
        for i, (tcol, bitmap, hist, dom_t, corr) in enumerate(targets):
            d = arr[i]
            d.target, d.bitmap, d.hist_t = _address(tcol), _address(bitmap), _address(hist)
            d.dom_t, d.n_corr = dom_t, len(corr)
            for j, (ccol, cooc, dom_c, tau) in enumerate(corr):
                d.corr[j], d.cooc[j], d.dom_c[j], d.tau[j] = _address(ccol), _address(cooc), dom_c, tau
        self._call("dr_domain_prune", arr, len(targets), n_rows, n_total, beta, removed)

    # ---- repair base / tile ----------------------------------------------------------------------
    def gather_rows_masked(self, cols, bitmaps, rows, n, out, f64=False, null_out=None):
        """null_out (int32 codes only): int32 [K][words] that receives the NULL bitmap of every tile column."""
        if null_out is not None:
            assert not f64
            self._call("dr_gather_rows_masked_nulls", cols, bitmaps, len(cols), rows, n, out, null_out,
                       int(null_out.shape[1]))
            return
        self._call("dr_gather_rows_masked_f64" if f64 else "dr_gather_rows_masked", cols, bitmaps, len(cols), rows,
                   n, out)

    def tile_null_bitmap(self, tile, n, n_cols, col, out, f64=False):
        self._call("dr_tile_null_bitmap_f64" if f64 else "dr_tile_null_bitmap", tile, n, n_cols, col, out)

    def gather(self, col, rows, n, out, f64=False):
        self._call("dr_gather_f64" if f64 else "dr_gather_i32", col, rows, n, out)

    def tile_gather(self, tile, n_cols, col, drows, n, out, f64=False):
        self._call("dr_tile_gather_f64" if f64 else "dr_tile_gather_i32", tile, n_cols, col, drows, n, out)

    def lookup_sorted(self, sorted_rows, n_sorted, keys, n, out):
        self._call("dr_lookup_sorted", sorted_rows, n_sorted, keys, n, out)

    def forest_predict(self, forest_struct, tile, n_cols, ctile, n_ccols, cells, n_cells, target_col, out_margin=None):
        self._call("dr_forest_predict", byref(forest_struct), tile, n_cols, ctile, n_ccols, cells, n_cells, target_col,
                   out_margin)

    def forest_predict_ranked(self, forest_struct, tile, n_cols, cells, n_cells, target_col, out_margin=None):
        self._call("dr_forest_predict_ranked", byref(forest_struct), tile, n_cols, cells, n_cells, target_col,
                   out_margin)

    def gbdt_train(self, params, bins, n_bins, y_class, y_value, weight, init, workspace, out_nodes, out_counts):
        self._call("dr_gbdt_train", byref(params), bins, n_bins, y_class, y_value, weight,
                   (c_double * len(init))(*[float(v) for v in init]), workspace, workspace.numel(), out_nodes,
                   out_counts)

    def gbdt_workspace_bytes(self, n_rows, n_seq):
        return int(self.lib.dr_gbdt_workspace_bytes(n_rows, n_seq))

    def gbdt_train_ex(self, params, boost, bins, n_bins, y_class, y_value, weight, init, workspace, out_nodes,
                      out_counts):
        """dr_gbdt_train with boosting options: boost is a dr_gbdt_boost (its drop schedule arrays must stay
        alive for the call) or None."""
        self._call("dr_gbdt_train_ex", byref(params), None if boost is None else byref(boost), bins, n_bins, y_class,
                   y_value, weight, (c_double * len(init))(*[float(v) for v in init]), workspace, workspace.numel(),
                   out_nodes, out_counts)

    def gbdt_train_ex_workspace_bytes(self, n_rows, n_seq, n_drops):
        return int(self.lib.dr_gbdt_train_ex_workspace_bytes(n_rows, n_seq, n_drops))

    def tile_fill(self, tile, n_cols, col, cells, n_cells, value):
        self._call("dr_tile_fill_i32", tile, n_cols, col, cells, n_cells, value)

    def scatter(self, col, rows, vals, n, f64=False):
        self._call("dr_scatter_f64" if f64 else "dr_scatter_i32", col, rows, vals, n)

    def fd_map_build(self, x_col, x_mask, y_col, y_mask, n_rows, dom_x, lo, hi):
        self._call("dr_fd_map_build", x_col, x_mask, y_col, y_mask, n_rows, dom_x, lo, hi)

    def tile_lut_fill(self, tile, n_cols, x_col, y_col, cells, n_cells, lut, lut_size):
        self._call("dr_tile_lut_fill", tile, n_cols, x_col, y_col, cells, n_cells, lut, lut_size)

    # ---- delphi.misc ------------------------------------------------------------------------------
    def kmeans_assign(self, cols, dom, p_off, n_rows, P, mu_sq, labels, split=None):
        """One k-means assignment over dictionary codes: P device float64 [p_rows][n_centres], mu_sq device
        float64 [n_centres]; labels device int32, written in place (only rows split[label] >= 0 with split)."""
        self._call("dr_kmeans_assign", cols, dom, p_off, len(cols), n_rows, P, int(P.shape[0]), mu_sq,
                   int(P.shape[1]), split, 0 if split is None else int(split.numel()), labels)

    def label_counts(self, labels, col, dom, n_rows, lab_lo, lab_hi, out):
        """out (device int64 [lab_hi - lab_lo][dom + 1], zeroed) += counts of (label, code slot)."""
        self._call("dr_label_counts", labels, col, dom, n_rows, lab_lo, lab_hi, out)

    def error_map(self, bitmaps, n_rows, out):
        self._call("dr_error_map", bitmaps, len(bitmaps), n_rows, out)

    def null_bits(self, valid, bit_offset, n_rows, row_base, key, ratio, out):
        self._call("dr_null_bits", valid, bit_offset, n_rows, row_base, key & ((1 << 64) - 1), float(ratio), out)

    def flatten(self, cols, base, n_rows, row_ids, out_codes, out_valid, out_ids):
        self._call("dr_flatten", cols, base, len(cols), n_rows, row_ids, out_codes, out_valid, out_ids)

    # ---- Spark-compatible distinct counts ---------------------------------------------------------------
    def hll_dict(self, kind, data, offsets, n, regs, hashes=None):
        """regs (device int32[512]) <- HLL++ registers of n dictionary entries; hashes (device uint64[n])
        receives each entry's seed-42 hash when given."""
        self._call("dr_hll_dict", kind, data, offsets, n, hashes, regs)

    def hll_pairs(self, pairs):
        """pairs: [(hx, y_kind, y_data, y_off, dom_x, dom_y, bits, regs)], buffers as tensors or addresses."""
        arr = (dr_hll_pair * max(len(pairs), 1))()
        for d, (hx, y_kind, y_data, y_off, dom_x, dom_y, bits, regs) in zip(arr, pairs):
            d.hx, d.y_data, d.y_off = _address(hx), _address(y_data), _address(y_off)
            d.bits, d.regs = _address(bits), _address(regs)
            d.dom_x, d.dom_y, d.y_kind = dom_x, dom_y, y_kind
        self._call("dr_hll_pairs", arr, len(pairs))


def _profiled(name, fn):
    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        if self.profile is None:
            return fn(self, *args, **kwargs)
        import torch
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        try:
            return fn(self, *args, **kwargs)
        finally:
            end.record()
            self.profile.append((name, start, end))
    return wrapper


# The public methods that do no device work; every other one records one profile entry per call, under its name.
_NOT_PROFILED = {"close", "acquire", "release", "launch_count", "gbdt_workspace_bytes"}
for _name, _fn in list(vars(Context).items()):
    if not _name.startswith("_") and _name not in _NOT_PROFILED:
        setattr(Context, _name, _profiled(_name, _fn))


def profile_summary(ctx):
    """{call name: (count, total milliseconds)} of the calls recorded while ctx.profile was a list
    (CUDA events on the launching stream)."""
    import torch
    torch.cuda.synchronize()
    out = {}
    for name, start, end in ctx.profile or []:
        c, t = out.get(name, (0, 0.0))
        out[name] = (c + 1, t + start.elapsed_time(end))
    return out
