"""ctypes binding of libannlite_b200.so (include/annb.h).

There is no CPU fallback anywhere in this package: if the shared library is missing the import of
any compute entry point raises, and the library itself returns ANNB_ENODEVICE without a GPU.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('ANNB_LIB_PATH') or os.path.join(_HERE, 'lib', 'libannlite_b200.so')   # the override is for A/B runs of kernel variants

OK, EINVAL, ENODEVICE, ECUDA, ENOMEM, ESTATE, EFEWRESULTS, EIO, ECAPACITY, ENOTFOUND, ELIMIT = (
    0, -1, -2, -3, -4, -5, -6, -7, -8, -9, -10)
HOST, DEVICE = 0, 1
METRIC_L2, METRIC_IP, METRIC_COSINE = 0, 1, 2
MAX_EF = 512
MAX_CELLS, CELLS_GENERIC, CELLS_EXACT = 256, 1, 2
ATTR_INTEGER, ATTR_FLOAT, ATTR_TEXT = 0, 1, 2
MAX_ATTR_COLUMNS, FILTER_MAX_OPS, FILTER_MAX_DEPTH, FILTER_MAX_CONST_BYTES = 64, 256, 32, 32768
FILTER_MAX_PER_CALL, FILTER_LAUNCH_MAX_OPS, FILTER_LAUNCH_MAX_CONST_BYTES = 1024, 2048, 65536
(FOP_FALSE, FOP_TRUE, FOP_NOTNULL, FOP_INT_RANGE, FOP_INT_NE, FOP_INT_IN, FOP_INT_NIN, FOP_FLT_RANGE, FOP_FLT_NE,
 FOP_FLT_IN, FOP_FLT_NIN, FOP_CODE_IN, FOP_AND, FOP_OR) = range(14)
# annb_filter_op_t
FILTER_OP = np.dtype([('op', '<i4'), ('col', '<i4'), ('a', '<i4'), ('b', '<i4')])
# annb_device_graph_export parts and header size
GRAPH_PARTS = ('header', 'rec0', 'upper', 'labels', 'deleted', 'wide_codes', 'own_codes')
GRAPH_MAX_LEVELS = 32
GRAPH_HEADER_BYTES = (14 + GRAPH_MAX_LEVELS) * 8 + 128

_lib = None

_i64, _u64, _i32, _u32, _int, _f64 = C.c_int64, C.c_uint64, C.c_int32, C.c_uint32, C.c_int, C.c_double
_vp, _cp = C.c_void_p, C.c_char_p

# name -> (restype, argtypes); kept in one table so tests can check it against include/annb.h
PROTOTYPES = {
    'annb_version': (_int, []),
    'annb_last_error': (_cp, []),
    'annb_device_count': (_int, []),
    'annb_create': (_int, [_int, _int, _int, _int, _int, C.POINTER(_vp)]),
    'annb_destroy': (_int, [_vp]),
    'annb_set_codebook': (_int, [_vp, _vp, _int]),
    'annb_stream': (_int, [_vp, C.POINTER(_u64)]),
    'annb_sync': (_int, [_vp]),
    'annb_adc_table': (_int, [_vp, _vp, _int, _i64, _int, _vp, _int]),
    'annb_set_codes': (_int, [_vp, _vp, _int, _i64]),
    'annb_scan': (_int, [_vp, _vp, _int, _vp, _int]),
    'annb_scan_topk': (_int, [_vp, _vp, _vp, _int, _i64, _int, _vp, _vp, _int]),
    'annb_init_graph': (_int, [_vp, _i64, _int, _int, _u64]),
    'annb_load_index': (_int, [_vp, _cp, _i64]),
    'annb_save_index': (_int, [_vp, _cp]),
    'annb_set_graph': (_int, [_vp, _vp, _u64, _u64, _u64, _u64, _vp, _u64, _vp, _i64, _u64, _i64, _i64, _i32, _u32,
                              _int, _int, _int, _int, _f64]),
    'annb_graph_info': (_int, [_vp, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_u64), C.POINTER(_u64),
                               C.POINTER(_i32), C.POINTER(_u32), C.POINTER(_int), C.POINTER(_int),
                               C.POINTER(_int), C.POINTER(_int), C.POINTER(_f64)]),
    'annb_get_graph': (_int, [_vp, _vp, _vp, _vp]),
    'annb_add_items': (_int, [_vp, _vp, _vp, _vp, _i64, _int]),
    'annb_add_items_with_tables': (_int, [_vp, _vp, _vp, _vp, _i64, _int]),
    'annb_encode': (_int, [_vp, _vp, _int, _i64, _vp, _int]),
    'annb_resize_index': (_int, [_vp, _i64]),
    'annb_mark_deleted': (_int, [_vp, _u64]),
    'annb_unmark_deleted': (_int, [_vp, _u64]),
    'annb_element_count': (_int, [_vp, C.POINTER(_i64)]),
    'annb_get_labels': (_int, [_vp, _vp, _i64]),
    'annb_get_codes': (_int, [_vp, _vp, _i64, _vp]),
    'annb_search': (_int, [_vp, _vp, _vp, _int, _i64, _int, _int, _int, _vp, _int, _i64, _vp, _vp, _int, _vp]),
    'annb_scan_subset': (_int, [_vp, _vp, _int, _i64, _int, _int, _vp, _i64, _vp, _vp]),
    'annb_search_submit': (_int, [_vp, _vp, _int, _i64, _int, _int, _int, _vp, _vp, _int, C.POINTER(_int)]),
    'annb_search_submit_filtered': (_int, [_vp, _vp, _int, _i64, _int, _int, _int, _vp, _int, _i64, _vp, _vp, _int, C.POINTER(_int)]),
    'annb_search_wait': (_int, [_vp, _int]),
    'annb_attr_define': (_int, [_vp, _int, _int]),
    'annb_attr_set': (_int, [_vp, _int, _vp, _i64, _vp, _vp, _int]),
    'annb_attr_export': (_int, [_vp, _int, _vp, _vp, _i64, C.POINTER(_i64)]),
    'annb_attr_clear': (_int, [_vp]),
    'annb_filter_prepare': (_int, [_vp, _vp, _int, _vp, _i64, C.POINTER(_int), C.POINTER(_i64)]),
    'annb_filter_labels': (_int, [_vp, _int, _vp, _i64, C.POINTER(_i64)]),
    'annb_filter_release': (_int, [_vp, _int]),
    'annb_filter_prepare_labels': (_int, [_vp, _vp, _i64, _int, C.POINTER(_int), C.POINTER(_i64)]),
    'annb_search_prepared': (_int, [_vp, _vp, _int, _i64, _int, _int, _int, _int, _vp, _vp, _int]),
    'annb_search_submit_prepared': (_int, [_vp, _vp, _int, _i64, _int, _int, _int, _int, _vp, _vp, _int, C.POINTER(_int)]),
    'annb_filter_prepare_many': (_int, [_vp, _int, _vp, _vp, _vp, _vp, _vp, _vp]),
    'annb_search_multi': (_int, [_vp, _vp, _int, _i64, _int, _int, _int, _vp, _vp, _vp, _int]),
    'annb_search_submit_multi': (_int, [_vp, _vp, _int, _i64, _int, _int, _int, _vp, _vp, _vp, _int, C.POINTER(_int)]),
    'annb_merge_topk': (_int,[_vp, _vp, _vp, _int, _i64, _int, _vp, _vp]),
    'annb_merge_topk_packed': (_int, [_vp, _vp, _int, _i64, _int, _i64, _i64, _vp, _vp, _int]),
    'annb_cellset_create': (_int, [_vp, _int, _vp, _int, C.POINTER(_vp)]),
    'annb_cellset_destroy': (_int, [_vp]),
    'annb_cellset_search': (_int, [_vp, _vp, _int, _i64, _int, _vp, _int, _int, _int, _int, _vp, _vp, _vp, _int, _vp, _vp, _vp]),
    'annb_cellset_search_prepared': (_int, [_vp, _vp, _int, _i64, _int, _vp, _int, _int, _int, _int, _vp, _vp, _vp, _vp, _int,
                                            _vp, _vp, _vp]),
    'annb_cellset_search_multi': (_int, [_vp, _vp, _int, _i64, _int, _vp, _int, _int, _int, _int, _vp, _vp, _vp, _vp, _int,
                                         _vp, _vp, _vp]),
    'annb_cellset_last_filtered': (_int, [_vp, C.POINTER(_i64), C.POINTER(_int)]),
    'annb_cellset_set_bruteforce': (_int, [_vp, _vp]),
    'annb_cellset_add_items': (_int, [_vp, _vp, _vp, _vp, _i64, _int]),
    'annb_cellset_last_build': (_int, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(_i64), C.POINTER(_int)]),
    'annb_cellset_last_scanned': (_int, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    'annb_cellset_merge': (_int, [_vp, _vp, _vp, _vp, _vp, _int, _i64, _int, _int, _vp, _vp, _vp, _int]),
    'annb_cellset_probe': (_int, [_vp, _vp, _int, _i64, _int, _vp, _int]),
    'annb_cellset_last_ms': (_int, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(_int)]),
    'annb_lane_stream': (_int, [_vp, _int, C.POINTER(_u64)]),
    'annb_last_kernel_ms': (_int, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    'annb_launch_count': (_int, [_vp, C.POINTER(_i64)]),
    'annb_fallback_count': (_int, [_vp, C.POINTER(_i64)]),
    'annb_fallback_queries': (_int, [_vp, C.POINTER(_i64)]),
    'annb_sync_counts': (_int, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    'annb_device_graph_layout': (_int, [_vp, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_int)]),
    'annb_device_graph_export': (_int, [_vp, _int, _vp, _i64, C.POINTER(_i64)]),
    'annb_set_option': (_int, [_vp, _cp, _i64]),
}


def load():
    """Load the shared library (once).  Raises if it has not been built: no silent fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                f'or `bash annlite_b200/csrc/build.sh`. annlite_b200 has no CPU fallback.')
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


class AnnbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


def check(rc):
    """Map a status code to the exception type the reference raises for the same condition."""
    if rc == OK:
        return
    msg = load().annb_last_error().decode('utf-8', 'replace')
    if rc == EINVAL:
        # a bad codec geometry, and a batch with a NaN or an infinity (scipy.cluster.vq's ValueError in the reference)
        refused = 'Initialization Error' in msg or 'must not contain infs or NaNs' in msg
        raise ValueError(msg) if refused else AnnbError(rc, msg)
    if rc == ENOMEM:
        raise MemoryError(msg)
    if rc == ELIMIT and 'PQ clustering exceed' in msg:
        raise ValueError(msg)
    raise AnnbError(rc, msg)   # RuntimeError subclass == what pybind11 turns std::runtime_error into


def as_ptr(x):
    """(pointer, space, keepalive) for a numpy array (host) or a torch CUDA tensor (device)."""
    if x is None:
        return None, HOST, None
    if isinstance(x, np.ndarray):
        if not x.flags['C_CONTIGUOUS']:
            x = np.ascontiguousarray(x)
        return x.ctypes.data, HOST, x
    if hasattr(x, 'data_ptr'):  # torch tensor
        if not x.is_contiguous():
            x = x.contiguous()
        return x.data_ptr(), (DEVICE if x.is_cuda else HOST), x
    raise TypeError(f'expected numpy array or torch tensor, got {type(x)}')
