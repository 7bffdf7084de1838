"""ctypes binding of the C ABI in include/lightctr_b200.h (lightctr_b200/lib/liblightctr_b200.so).

This is plumbing for the Python tests and bench.py; the drop-in host side for the reference's C++
callers is lightctr_b200/host/*.h.  There is NO CPU fallback: if the shared library is missing or
no CUDA device is present the calls raise.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "liblightctr_b200.so")

MODEL_FM, MODEL_FFM, MODEL_NFM, MODEL_WND = 1, 2, 3, 4
OPT_ADAGRAD, OPT_FTRL, OPT_ADAM, OPT_RMSPROP, OPT_ADADELTA = 0, 1, 2, 3, 4
PIPE_DEPTH = 3  # LCTR_PIPE_DEPTH: tickets of train_batch_async that may be outstanding
OPT_PS_SGD, OPT_PS_ADAGRAD, OPT_PS_DCASGD, OPT_PS_DCASGDA = 5, 6, 7, 8
ACT_SIGMOID, ACT_TANH = 0, 1
MLP_FP32, MLP_BF16 = 0, 1
KEYS_DENSE, KEYS_HASHED = 0, 1
RESERVED_KEY = (1 << 64) - 1  # the key table's empty marker: never a valid key
MAX_LAYERS = 8
ABI_VERSION = 1

# every symbol include/lightctr_b200.h declares (tests check the .so exports each of them)
SYMBOLS = [
    "lctr_last_error", "lctr_abi_version", "lctr_create", "lctr_destroy", "lctr_sync", "lctr_upload_params",
    "lctr_download_params", "lctr_fill_params", "lctr_download_opt_state", "lctr_upload_opt_state", "lctr_upload_batch",
    "lctr_train_step", "lctr_train_batch", "lctr_train_batch_async", "lctr_wait", "lctr_predict", "lctr_score", "lctr_download_sumvx", "lctr_download_pred",
    "lctr_mlp_forward", "lctr_mlp_backward", "lctr_mlp_apply", "lctr_mlp_upload", "lctr_mlp_download", "lctr_mlp_set_mask", "lctr_mlp_download_grad", "lctr_set_dense_allreduce", "lctr_save_checkpoint", "lctr_load_checkpoint",
    "lctr_save_dataset_bin", "lctr_load_dataset_bin", "lctr_eval", "lctr_upload_pred", "lctr_ipc_export", "lctr_ipc_import",
    "lctr_dense_grad_buffer", "lctr_device_bytes", "lctr_load_libffm", "lctr_free_dataset", "lctr_launch_count", "lctr_stream", "lctr_profile", "lctr_profile_read",
    "lctr_upload_batch_keys", "lctr_lookup_keys", "lctr_download_keys", "lctr_upload_keyed_params", "lctr_set_key_init",
    "lctr_load_libffm_keys", "lctr_free_keyed_dataset", "lctr_evict_keys", "lctr_load_checkpoint_shards", "lctr_eval_pred",
    "lctr_download_host_tier", "lctr_evict_host_tier", "lctr_set_key_admission", "lctr_decay_key_admission",
    "lctr_key_admission_stats", "lctr_upload_libffm", "lctr_download_batch", "lctr_track_changes", "lctr_save_checkpoint_delta",
    "lctr_load_checkpoint_chain", "lctr_checkpoint_hash", "lctr_set_row_weights", "lctr_train_batch_weighted_async",
    "lctr_eval_weighted", "lctr_eval_pred_weighted",
]
NO_LIMIT = (1 << 64) - 1  # lctr_evict_keys: UINT64_MAX = no limit
TEXT_BEGIN, TEXT_END, TEXT_LOOKUP = 1, 2, 4  # lctr_upload_libffm flags


class Cfg(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("model", C.c_int32), ("optimizer", C.c_int32), ("device", C.c_int32),
                ("feature_cnt", C.c_uint64), ("field_cnt", C.c_uint32), ("factor_cnt", C.c_uint32),
                ("learning_rate", C.c_float), ("l2_reg", C.c_float), ("minibatch_size", C.c_uint64),
                ("momentum", C.c_float), ("momentum_adam2", C.c_float), ("ftrl_alpha", C.c_float),
                ("ftrl_beta", C.c_float), ("ftrl_lambda1", C.c_float), ("ftrl_lambda2", C.c_float),
                ("n_hidden", C.c_int32), ("hidden", C.c_uint32 * MAX_LAYERS), ("activation", C.c_int32),
                ("mlp_precision", C.c_int32), ("max_rows", C.c_uint64), ("max_nnz", C.c_uint64), ("rank", C.c_int32),
                ("world", C.c_int32), ("deterministic", C.c_int32), ("key_mode", C.c_int32),
                ("csc_row_block", C.c_uint64), ("ema_rate", C.c_float), ("key_evict", C.c_int32),
                ("reserved", C.c_uint32 * 2)]

    # cfg.key_host_rows shares its word with reserved[0] (a union in the header)
    key_host_rows = property(lambda self: self.reserved[0], lambda self, v: self.reserved.__setitem__(0, v))


class DatasetC(C.Structure):
    _fields_ = [("rows", C.c_int64), ("nnz", C.c_int64), ("label_cnt", C.c_int64), ("feature_cnt", C.c_uint64),
                ("field_cnt", C.c_uint64), ("row_ptr", C.POINTER(C.c_int64)), ("fid", C.POINTER(C.c_uint32)),
                ("field", C.POINTER(C.c_uint16)), ("val", C.POINTER(C.c_float)), ("label", C.POINTER(C.c_int32))]


class KeyedDatasetC(C.Structure):
    _fields_ = [("rows", C.c_int64), ("nnz", C.c_int64), ("label_cnt", C.c_int64), ("field_cnt", C.c_uint64),
                ("row_ptr", C.POINTER(C.c_int64)), ("key", C.POINTER(C.c_uint64)), ("field", C.POINTER(C.c_uint16)),
                ("val", C.POINTER(C.c_float)), ("label", C.POINTER(C.c_int32))]


class TextInfo(C.Structure):
    """lctr_text_info: what one lctr_upload_libffm call parsed"""
    _fields_ = [("rows", C.c_int64), ("nnz", C.c_int64), ("lines", C.c_int64), ("labels", C.c_int64),
                ("feature_cnt", C.c_uint64), ("field_cnt", C.c_uint64), ("host_lines", C.c_int64), ("consumed", C.c_size_t)]


_lib = None


def load_library():
    """dlopen the CUDA extension; raises loudly when it is missing (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("lightctr_b200: CUDA extension %s is missing -- run `python -m lightctr_b200.build` "
                           "(there is no CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i64, f32p = C.c_void_p, C.c_int64, C.c_void_p
    L.lctr_last_error.restype = C.c_char_p
    L.lctr_create.argtypes = [C.POINTER(Cfg), C.POINTER(vp)]
    L.lctr_destroy.argtypes = [vp]
    L.lctr_sync.argtypes = [vp]
    L.lctr_upload_params.argtypes = [vp, f32p, f32p]
    L.lctr_download_params.argtypes = [vp, f32p, f32p]
    L.lctr_fill_params.argtypes = [vp, C.c_uint64, C.c_float]
    L.lctr_download_opt_state.argtypes = [vp, f32p, f32p]
    L.lctr_upload_opt_state.argtypes = [vp, f32p, f32p]
    L.lctr_upload_batch.argtypes = [vp, C.c_int, i64, i64, vp, vp, vp, vp, vp]
    L.lctr_train_step.argtypes = [vp, C.c_int, i64, i64, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.lctr_set_row_weights.argtypes = [vp, C.c_int, i64, f32p]
    L.lctr_train_batch.argtypes = [vp, i64, i64, vp, vp, vp, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.lctr_train_batch_async.argtypes = [vp, i64, i64, vp, vp, vp, vp, vp, C.POINTER(C.c_uint64)]
    L.lctr_train_batch_weighted_async.argtypes = [vp, i64, i64, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_uint64)]
    L.lctr_wait.argtypes = [vp, C.c_uint64, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.lctr_predict.argtypes = [vp, C.c_int, C.c_int, f32p]
    L.lctr_score.argtypes = [vp, C.c_int, i64, i64, f32p]
    L.lctr_download_sumvx.argtypes = [vp, C.c_int, f32p]
    L.lctr_download_pred.argtypes = [vp, C.c_int, f32p]
    L.lctr_mlp_upload.argtypes = [vp, C.c_int, f32p, f32p]
    L.lctr_mlp_download.argtypes = [vp, C.c_int, f32p, f32p]
    L.lctr_mlp_set_mask.argtypes = [vp, C.c_int, f32p]
    L.lctr_mlp_forward.argtypes = [vp, i64, vp, vp]
    L.lctr_mlp_backward.argtypes = [vp, i64, vp, vp]
    L.lctr_mlp_apply.argtypes = [vp, C.c_uint64]
    L.lctr_mlp_download_grad.argtypes = [vp, C.c_int, f32p, f32p]
    L.lctr_set_dense_allreduce.argtypes = [vp, ALLREDUCE_FN, vp]
    L.lctr_eval.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int64), C.POINTER(C.c_float)]
    L.lctr_upload_pred.argtypes = [vp, C.c_int, f32p]
    L.lctr_eval_pred.argtypes = [vp, i64, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_int64), C.POINTER(C.c_float)]
    L.lctr_eval_weighted.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_float)]
    L.lctr_eval_pred_weighted.argtypes = [vp, i64, vp, vp, vp, C.POINTER(C.c_float), C.POINTER(C.c_double),
                                          C.POINTER(C.c_float)]
    L.lctr_save_checkpoint.argtypes = [vp, C.c_char_p]
    L.lctr_load_checkpoint.argtypes = [vp, C.c_char_p]
    L.lctr_load_checkpoint_shards.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p)]
    L.lctr_save_dataset_bin.argtypes = [C.POINTER(DatasetC), C.c_char_p]
    L.lctr_load_dataset_bin.argtypes = [C.c_char_p, C.POINTER(C.POINTER(DatasetC))]
    L.lctr_ipc_export.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    L.lctr_ipc_import.argtypes = [vp, vp, C.c_size_t]
    L.lctr_dense_grad_buffer.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.lctr_load_libffm.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(C.POINTER(DatasetC))]
    L.lctr_free_dataset.argtypes = [C.POINTER(DatasetC)]
    L.lctr_launch_count.argtypes = [vp]
    L.lctr_launch_count.restype = C.c_int64
    L.lctr_stream.argtypes = [vp]
    L.lctr_stream.restype = vp
    L.lctr_profile.argtypes = [vp, C.c_int]
    L.lctr_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int, C.c_int]
    L.lctr_upload_batch_keys.argtypes = [vp, C.c_int, i64, i64, vp, vp, vp, vp, vp, C.c_int]
    L.lctr_lookup_keys.argtypes = [vp, i64, vp, vp]
    L.lctr_download_keys.argtypes = [vp, vp, C.c_uint64, C.POINTER(C.c_uint64)]
    L.lctr_upload_keyed_params.argtypes = [vp, i64, vp, f32p, f32p]
    L.lctr_set_key_init.argtypes = [vp, C.c_uint64, C.c_float]
    L.lctr_load_libffm_keys.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.POINTER(KeyedDatasetC))]
    L.lctr_free_keyed_dataset.argtypes = [C.POINTER(KeyedDatasetC)]
    L.lctr_evict_keys.argtypes = [vp, C.c_uint64, C.c_uint64, vp, f32p, f32p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.lctr_evict_host_tier.argtypes = [vp, C.c_uint64, C.c_uint64, vp, f32p, f32p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.lctr_download_host_tier.argtypes = [vp, vp, f32p, f32p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.lctr_set_key_admission.argtypes = [vp, C.c_uint32, C.c_uint32]
    L.lctr_decay_key_admission.argtypes = [vp, C.c_uint32]
    L.lctr_key_admission_stats.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.lctr_upload_libffm.argtypes = [vp, C.c_int, vp, C.c_size_t, C.c_int, C.POINTER(TextInfo)]
    L.lctr_download_batch.argtypes = [vp, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64), vp, vp, vp, vp, vp]
    L.lctr_track_changes.argtypes = [vp, C.c_int]
    L.lctr_save_checkpoint_delta.argtypes = [vp, C.c_char_p, C.POINTER(C.c_uint64)]
    L.lctr_load_checkpoint_chain.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p)]
    L.lctr_checkpoint_hash.argtypes = [C.c_char_p, C.POINTER(C.c_uint64)]
    _lib = L
    return L


class LctrError(RuntimeError):
    pass


def _chk(rc):
    if rc != 0:
        raise LctrError(load_library().lctr_last_error().decode())


def _p(a):
    return None if a is None else a.ctypes.data


class HostDataset:
    """CSR arrays as produced by lctr_load_libffm (FM_Algo_Abst::dataSet / label)."""

    def __init__(self, row_ptr, fid, field, val, label, feature_cnt, field_cnt):
        self.row_ptr = np.ascontiguousarray(row_ptr, np.int64)
        self.fid = np.ascontiguousarray(fid, np.uint32)
        self.field = None if field is None else np.ascontiguousarray(field, np.uint16)
        self.val = None if val is None else np.ascontiguousarray(val, np.float32)
        self.label = np.ascontiguousarray(label, np.int32)
        self.feature_cnt, self.field_cnt = int(feature_cnt), int(field_cnt)

    rows = property(lambda self: len(self.row_ptr) - 1)
    nnz = property(lambda self: len(self.fid))


def load_libffm(path, field_cnt=0, feature_cnt=0):
    """FM_Algo_Abst::loadDataRow (fm_algo_abst.h:70-107) through the library's own parser."""
    L = load_library()
    dp = C.POINTER(DatasetC)()
    _chk(L.lctr_load_libffm(path.encode(), field_cnt, feature_cnt, C.byref(dp)))
    d = dp.contents
    n, r, lc = d.nnz, d.rows, d.label_cnt
    out = HostDataset(np.ctypeslib.as_array(d.row_ptr, (r + 1,)).copy(),
                      np.ctypeslib.as_array(d.fid, (max(n, 1),))[:n].copy(),
                      np.ctypeslib.as_array(d.field, (max(n, 1),))[:n].copy(),
                      np.ctypeslib.as_array(d.val, (max(n, 1),))[:n].copy(),
                      np.ctypeslib.as_array(d.label, (max(lc, 1),))[:lc].copy(), d.feature_cnt, d.field_cnt)
    L.lctr_free_dataset(dp)
    return out


class KeyedHostDataset:
    """CSR arrays as produced by lctr_load_libffm_keys: `key` holds the ids at their full 64-bit width."""

    def __init__(self, row_ptr, key, field, val, label, field_cnt):
        self.row_ptr = np.ascontiguousarray(row_ptr, np.int64)
        self.key = np.ascontiguousarray(key, np.uint64)
        self.field = None if field is None else np.ascontiguousarray(field, np.uint16)
        self.val = None if val is None else np.ascontiguousarray(val, np.float32)
        self.label = np.ascontiguousarray(label, np.int32)
        self.field_cnt = int(field_cnt)

    rows = property(lambda self: len(self.row_ptr) - 1)
    nnz = property(lambda self: len(self.key))


def load_libffm_keys(path, field_cnt=0):
    """The libffm parser of load_libffm with 64-bit ids, for keyed contexts."""
    L = load_library()
    dp = C.POINTER(KeyedDatasetC)()
    _chk(L.lctr_load_libffm_keys(path.encode(), field_cnt, C.byref(dp)))
    d = dp.contents
    n, r, lc = d.nnz, d.rows, d.label_cnt
    out = KeyedHostDataset(np.ctypeslib.as_array(d.row_ptr, (r + 1,)).copy(),
                           np.ctypeslib.as_array(d.key, (max(n, 1),))[:n].copy(),
                           np.ctypeslib.as_array(d.field, (max(n, 1),))[:n].copy(),
                           np.ctypeslib.as_array(d.val, (max(n, 1),))[:n].copy(),
                           np.ctypeslib.as_array(d.label, (max(lc, 1),))[:lc].copy(), d.field_cnt)
    L.lctr_free_keyed_dataset(dp)
    return out


def _dataset_from_c(d):
    n, r, lc = d.nnz, d.rows, d.label_cnt
    return HostDataset(np.ctypeslib.as_array(d.row_ptr, (r + 1,)).copy(),
                       np.ctypeslib.as_array(d.fid, (max(n, 1),))[:n].copy(),
                       np.ctypeslib.as_array(d.field, (max(n, 1),))[:n].copy(),
                       np.ctypeslib.as_array(d.val, (max(n, 1),))[:n].copy(),
                       np.ctypeslib.as_array(d.label, (max(lc, 1),))[:lc].copy(), d.feature_cnt, d.field_cnt)


def libffm_to_bin(path, bin_path, field_cnt=0, feature_cnt=0):
    """Parse a libffm text file once and write the binary CSR cache next to it."""
    L = load_library()
    dp = C.POINTER(DatasetC)()
    _chk(L.lctr_load_libffm(path.encode(), field_cnt, feature_cnt, C.byref(dp)))
    try:
        _chk(L.lctr_save_dataset_bin(dp, bin_path.encode()))
    finally:
        L.lctr_free_dataset(dp)


def load_dataset_bin(bin_path):
    L = load_library()
    dp = C.POINTER(DatasetC)()
    _chk(L.lctr_load_dataset_bin(bin_path.encode(), C.byref(dp)))
    out = _dataset_from_c(dp.contents)
    L.lctr_free_dataset(dp)
    return out


def checkpoint_hash(path):
    """the 64-bit hash that links an incremental checkpoint to its parent, of any file (host only)"""
    h = C.c_uint64()
    _chk(load_library().lctr_checkpoint_hash(path.encode(), C.byref(h)))
    return h.value


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)


class Context:
    """Owning wrapper around lctr_ctx."""

    def __init__(self, model, feature_cnt, factor_cnt, field_cnt=0, optimizer=OPT_ADAGRAD, lr=0.05, l2=0.001,
                 minibatch_size=0, momentum=0.8, momentum_adam2=0.999, hidden=(), activation=ACT_SIGMOID,
                 mlp_precision=MLP_FP32, device=0, rank=0, world=1, deterministic=0, csc_row_block=0, max_rows=0,
                 max_nnz=0, ema_rate=0.99, key_mode=KEYS_DENSE, key_evict=False, key_host_rows=0):
        """key_mode=KEYS_HASHED: batches carry uint64 keys (upload_batch_keys) and feature_cnt is the row capacity.
        key_evict=True (keyed only): rows record the insert-upload that last met them, for evict_keys.
        key_host_rows > 0 (with key_evict=True): evicted rows go to a host-memory tier of that many rows and come back
        when their keys do."""
        L = load_library()
        cfg = Cfg()
        cfg.abi_version = ABI_VERSION
        cfg.model, cfg.optimizer, cfg.device = model, optimizer, device
        cfg.feature_cnt, cfg.field_cnt, cfg.factor_cnt = feature_cnt, field_cnt, factor_cnt
        cfg.learning_rate, cfg.l2_reg, cfg.minibatch_size = lr, l2, minibatch_size
        cfg.momentum, cfg.momentum_adam2 = momentum, momentum_adam2
        cfg.ema_rate = ema_rate
        cfg.n_hidden = len(hidden)
        for i, h in enumerate(hidden):
            cfg.hidden[i] = h
        cfg.activation, cfg.mlp_precision = activation, mlp_precision
        cfg.rank, cfg.world = rank, world
        cfg.deterministic, cfg.csc_row_block = deterministic, csc_row_block
        cfg.max_rows, cfg.max_nnz = max_rows, max_nnz
        cfg.key_mode = key_mode
        cfg.key_evict = 1 if key_evict else 0
        cfg.key_host_rows = key_host_rows
        self.cfg = cfg
        self.h = C.c_void_p()
        _chk(L.lctr_create(C.byref(cfg), C.byref(self.h)))
        self.L = L
        self.F, self.k, self.Fc = feature_cnt, factor_cnt, field_cnt
        self.rowlen = factor_cnt * (field_cnt if model == MODEL_FFM else 1)
        self.slot_rows = {}

    def close(self):
        if self.h:
            self.L.lctr_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        _chk(self.L.lctr_sync(self.h))

    def upload_params(self, W, V):
        W = None if W is None else np.ascontiguousarray(W, np.float32)
        V = None if V is None else np.ascontiguousarray(V, np.float32)
        _chk(self.L.lctr_upload_params(self.h, _p(W), _p(V)))

    def fill_params(self, seed, scale):
        _chk(self.L.lctr_fill_params(self.h, seed, scale))

    def download_params(self):
        W = np.empty(self.F, np.float32)
        V = np.empty(self.F * self.rowlen, np.float32)
        _chk(self.L.lctr_download_params(self.h, W.ctypes.data, V.ctypes.data))
        return W, V

    def download_opt_state(self):
        n = self.F * (self.rowlen + 1)
        s1, s2 = np.zeros(n, np.float32), np.zeros(n, np.float32)
        _chk(self.L.lctr_download_opt_state(self.h, s1.ctypes.data, s2.ctypes.data))
        return s1, s2

    def upload_opt_state(self, s1, s2=None):
        s1 = np.ascontiguousarray(s1, np.float32)
        s2 = None if s2 is None else np.ascontiguousarray(s2, np.float32)
        _chk(self.L.lctr_upload_opt_state(self.h, _p(s1), _p(s2)))

    def upload_batch(self, slot, row_ptr, fid, field, val, label):
        rows, nnz = len(row_ptr) - 1, len(fid)
        keep = [np.ascontiguousarray(row_ptr, np.int64), np.ascontiguousarray(fid, np.uint32),
                None if field is None else np.ascontiguousarray(field, np.uint16),
                None if val is None else np.ascontiguousarray(val, np.float32), np.ascontiguousarray(label, np.int32)]
        _chk(self.L.lctr_upload_batch(self.h, slot, rows, nnz, *[_p(a) for a in keep]))
        self.sync()  # host arrays may be pageable temporaries
        self.slot_rows[slot] = rows

    def upload_batch_keys(self, slot, row_ptr, key, field, val, label, insert=True):
        """keyed twin of upload_batch: key (uint64) per entry; insert=False maps unseen keys to the null row"""
        rows, nnz = len(row_ptr) - 1, len(key)
        keep = [np.ascontiguousarray(row_ptr, np.int64), np.ascontiguousarray(key, np.uint64),
                None if field is None else np.ascontiguousarray(field, np.uint16),
                None if val is None else np.ascontiguousarray(val, np.float32), np.ascontiguousarray(label, np.int32)]
        self.slot_rows[slot] = 0
        _chk(self.L.lctr_upload_batch_keys(self.h, slot, rows, nnz, *[_p(a) for a in keep], 1 if insert else 0))
        self.sync()
        self.slot_rows[slot] = rows

    def lookup_keys(self, keys):
        """row of each key (int64), -1 where absent"""
        k = np.ascontiguousarray(keys, np.uint64)
        out = np.empty(len(k), np.int64)
        _chk(self.L.lctr_lookup_keys(self.h, len(k), _p(k), _p(out)))
        return out

    def download_keys(self):
        """row -> key map (uint64) of the rows in use"""
        n = C.c_uint64()
        _chk(self.L.lctr_download_keys(self.h, None, 0, C.byref(n)))
        out = np.empty(n.value, np.uint64)
        _chk(self.L.lctr_download_keys(self.h, _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def upload_keyed_params(self, keys, W=None, V=None):
        k = np.ascontiguousarray(keys, np.uint64)
        W = None if W is None else np.ascontiguousarray(W, np.float32)
        V = None if V is None else np.ascontiguousarray(V, np.float32)
        _chk(self.L.lctr_upload_keyed_params(self.h, len(k), _p(k), _p(W), _p(V)))

    def set_key_init(self, seed, scale):
        _chk(self.L.lctr_set_key_init(self.h, seed, scale))

    def evict_keys(self, max_idle=None, max_rows=None, export=False):
        """Free rows idle for more than max_idle insert-uploads, then the oldest beyond max_rows (None = no limit).
        Returns the number evicted, or with export=True (keys, W, V) of the evicted rows in ascending order of their
        old row (V flat, rowlen floats per key)."""
        idle = NO_LIMIT if max_idle is None else int(max_idle)
        rows = NO_LIMIT if max_rows is None else int(max_rows)
        n = C.c_uint64()
        if not export:
            _chk(self.L.lctr_evict_keys(self.h, idle, rows, None, None, None, 0, C.byref(n)))
            return n.value
        cap = len(self.download_keys())  # at most the rows in use can leave
        keys = np.empty(max(cap, 1), np.uint64)
        W = np.empty(max(cap, 1), np.float32)
        V = np.empty(max(cap, 1) * self.rowlen, np.float32)
        _chk(self.L.lctr_evict_keys(self.h, idle, rows, _p(keys), _p(W), _p(V), cap, C.byref(n)))
        m = n.value
        return keys[:m].copy(), W[:m].copy(), V[:m * self.rowlen].copy()

    def download_host_tier(self):
        """(keys, W, V) of the host tier's rows in tier order (V flat, rowlen floats per key)"""
        n = C.c_uint64()
        _chk(self.L.lctr_download_host_tier(self.h, None, None, None, 0, C.byref(n)))
        m = n.value
        keys, W, V = np.empty(max(m, 1), np.uint64), np.empty(max(m, 1), np.float32), np.empty(max(m, 1) * self.rowlen, np.float32)
        _chk(self.L.lctr_download_host_tier(self.h, _p(keys), _p(W), _p(V), m, C.byref(n)))
        return keys[:m].copy(), W[:m].copy(), V[:m * self.rowlen].copy()

    def evict_host_tier(self, max_idle=None, max_rows=None, export=False):
        """evict_keys's rule on the host tier's rows; the rows it frees leave the model.  Returns the number freed, or
        with export=True (keys, W, V) of the freed rows in ascending order of their tier row."""
        idle = NO_LIMIT if max_idle is None else int(max_idle)
        rows = NO_LIMIT if max_rows is None else int(max_rows)
        n = C.c_uint64()
        if not export:
            _chk(self.L.lctr_evict_host_tier(self.h, idle, rows, None, None, None, 0, C.byref(n)))
            return n.value
        _chk(self.L.lctr_download_host_tier(self.h, None, None, None, 0, C.byref(n)))
        cap = n.value
        keys = np.empty(max(cap, 1), np.uint64)
        W = np.empty(max(cap, 1), np.float32)
        V = np.empty(max(cap, 1) * self.rowlen, np.float32)
        _chk(self.L.lctr_evict_host_tier(self.h, idle, rows, _p(keys), _p(W), _p(V), cap, C.byref(n)))
        m = n.value
        return keys[:m].copy(), W[:m].copy(), V[:m * self.rowlen].copy()

    def set_key_admission(self, min_count, log2_width=20):
        """Give a new key a row only once insert-uploads have met it min_count times, counted in a count-min sketch of
        4 x 2^log2_width counters (zeroed by this call); min_count <= 1 turns admission off.  Entries of keys not admitted
        are dropped from the batch, rows stay."""
        _chk(self.L.lctr_set_key_admission(self.h, int(min_count), int(log2_width)))

    def decay_key_admission(self, shift):
        """every counter of the admission sketch >>= shift (1..32)"""
        _chk(self.L.lctr_decay_key_admission(self.h, int(shift)))

    def key_admission_stats(self):
        """(entries dropped, keys admitted) by the last insert-upload"""
        d, a = C.c_uint64(), C.c_uint64()
        _chk(self.L.lctr_key_admission_stats(self.h, C.byref(d), C.byref(a)))
        return d.value, a.value

    def upload_libffm(self, slot, data, begin=True, end=True, lookup=False):
        """libffm text (bytes or any buffer; pinned memory copies fastest) parsed into `slot` on the device -> TextInfo.
        Consecutive calls continue one file: begin=True on its first part, end=True on its last."""
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        flags = (TEXT_BEGIN if begin else 0) | (TEXT_END if end else 0) | (TEXT_LOOKUP if lookup else 0)
        info = TextInfo()
        self.slot_rows[slot] = 0
        _chk(self.L.lctr_upload_libffm(self.h, slot, buf.ctypes.data, len(data), flags, C.byref(info)))
        self.slot_rows[slot] = info.rows
        return info

    def download_batch(self, slot):
        """the slot read back -> (row_ptr, fid, field, val, label): fid holds table rows on keyed contexts, val is 1.0f
        where the slot stores none, label the floats the slot trains on"""
        rows, nnz = C.c_int64(), C.c_int64()
        _chk(self.L.lctr_download_batch(self.h, slot, C.byref(rows), C.byref(nnz), None, None, None, None, None))
        r, n = rows.value, nnz.value
        row_ptr, fid, field = np.empty(r + 1, np.int64), np.empty(n, np.uint32), np.empty(n, np.uint16)
        val, label = np.empty(n, np.float32), np.empty(r, np.float32)
        _chk(self.L.lctr_download_batch(self.h, slot, None, None, *[a.ctypes.data for a in (row_ptr, fid, field, val, label)]))
        return row_ptr, fid, field, val, label

    def upload_dataset(self, slot, ds, all_ones_as_null=True):
        val = ds.val
        if val is not None and all_ones_as_null and np.all(val == 1.0):
            val = None
        self.upload_batch(slot, ds.row_ptr, ds.fid, ds.field, val, ds.label[:len(ds.row_ptr) - 1])

    def set_row_weights(self, slot, weights):
        """Per-row weights (float32, one per row of the batch in `slot`) for the train steps on that batch; None drops
        them.  Any later upload into the slot drops them too (include/lightctr_b200.h states the rule)."""
        if weights is None:
            _chk(self.L.lctr_set_row_weights(self.h, slot, 0, None))
            return
        w = np.ascontiguousarray(weights, np.float32)
        _chk(self.L.lctr_set_row_weights(self.h, slot, len(w), _p(w)))

    def train_step(self, slot=0, row_begin=0, row_end=None, want_stats=True):
        if row_end is None:
            row_end = self.slot_rows[slot]
        if want_stats:
            loss, acc = C.c_float(), C.c_float()
            _chk(self.L.lctr_train_step(self.h, slot, row_begin, row_end, C.byref(loss), C.byref(acc)))
            return loss.value, acc.value
        _chk(self.L.lctr_train_step(self.h, slot, row_begin, row_end, None, None))
        return None

    def train_batch(self, row_ptr, fid, field, val, label):
        """End-to-end call on host buffers (numpy arrays, ideally pinned)."""
        loss, acc = C.c_float(), C.c_float()
        _chk(self.L.lctr_train_batch(self.h, len(row_ptr) - 1, len(fid), _p(row_ptr), _p(fid), _p(field), _p(val),
                                     _p(label), C.byref(loss), C.byref(acc)))
        return loss.value, acc.value

    def train_batch_async(self, row_ptr, fid, field, val, label, weight=None):
        """Streamed step on host buffers; returns the ticket for wait().  weight (float32, one per row) trains the batch
        weighted (lctr_train_batch_weighted_async).  Every buffer must stay alive until the ticket has been waited for."""
        t = C.c_uint64()
        if weight is None:
            _chk(self.L.lctr_train_batch_async(self.h, len(row_ptr) - 1, len(fid), _p(row_ptr), _p(fid), _p(field), _p(val),
                                               _p(label), C.byref(t)))
            return t.value
        if len(weight) != len(row_ptr) - 1:
            raise ValueError("train_batch_async: %d weights for %d rows" % (len(weight), len(row_ptr) - 1))
        _chk(self.L.lctr_train_batch_weighted_async(self.h, len(row_ptr) - 1, len(fid), _p(row_ptr), _p(fid), _p(field),
                                                    _p(val), _p(label), _p(weight), C.byref(t)))
        return t.value

    def wait(self, ticket):
        loss, acc = C.c_float(), C.c_float()
        _chk(self.L.lctr_wait(self.h, ticket, C.byref(loss), C.byref(acc)))
        return loss.value, acc.value

    def predict(self, slot, quirk_sumvx_slot=-1):
        out = np.empty(self.slot_rows[slot], np.float32)
        _chk(self.L.lctr_predict(self.h, slot, quirk_sumvx_slot, out.ctypes.data))
        return out

    def predict_resident(self, slot, quirk_sumvx_slot=-1):
        """forward only, predictions stay on the device (no host copy, no synchronisation)"""
        _chk(self.L.lctr_predict(self.h, slot, quirk_sumvx_slot, None))

    def score(self, slot, row_begin=0, row_end=None, download=True):
        """the pCTR a train step on rows [row_begin, row_end) would compute, bit for bit, with no side effects (they are
        also left in the slot's pred array); download=False keeps them on the device (no copy, no synchronisation)"""
        if row_end is None:
            row_end = self.slot_rows[slot]
        if not download:
            _chk(self.L.lctr_score(self.h, slot, row_begin, row_end, None))
            return None
        out = np.empty(max(row_end - row_begin, 0), np.float32)
        _chk(self.L.lctr_score(self.h, slot, row_begin, row_end, out.ctypes.data))
        return out

    def download_sumvx(self, slot):
        out = np.empty(self.slot_rows[slot] * self.k, np.float32)
        _chk(self.L.lctr_download_sumvx(self.h, slot, out.ctypes.data))
        return out

    def download_pred(self, slot):
        out = np.empty(self.slot_rows[slot], np.float32)
        _chk(self.L.lctr_download_pred(self.h, slot, out.ctypes.data))
        return out

    def mlp_upload(self, layer, weight, bias):
        w = np.ascontiguousarray(weight, np.float32)
        b = np.ascontiguousarray(bias, np.float32)
        _chk(self.L.lctr_mlp_upload(self.h, layer, w.ctypes.data, b.ctypes.data))

    def mlp_download(self, layer, n_in, n_out):
        w, b = np.empty(n_in * n_out, np.float32), np.empty(n_out, np.float32)
        _chk(self.L.lctr_mlp_download(self.h, layer, w.ctypes.data, b.ctypes.data))
        return w, b

    def set_dense_allreduce(self, fn):
        """fn(dev_ptr:int, n_floats:int, cuda_stream:int) -> None: in-place SUM all-reduce enqueued on that stream."""
        def tramp(user, buf, n, stream):
            try:
                fn(buf, n, stream or 0)
                return 0
            except Exception:  # exceptions must not cross the C boundary
                import traceback
                traceback.print_exc()
                return 1
        self._allreduce_cb = ALLREDUCE_FN(tramp)  # keep alive
        _chk(self.L.lctr_set_dense_allreduce(self.h, self._allreduce_cb, None))

    def eval_metrics(self, slot):
        """(summed logloss, correct count, AUC) of the slot's pCTR / labels, computed on the device."""
        loss, correct, auc = C.c_float(), C.c_int64(), C.c_float()
        _chk(self.L.lctr_eval(self.h, slot, C.byref(loss), C.byref(correct), C.byref(auc)))
        return loss.value, correct.value, auc.value

    def eval_pred(self, pctr, labels, weights=None):
        """eval_metrics over host arrays: (summed logloss, correct count, AUC) of pctr against labels, in row order.  With
        weights (one per row) the weighted metrics of lctr_eval_pred_weighted, the correct count then a float."""
        p = np.ascontiguousarray(pctr, np.float32)
        y = np.ascontiguousarray(labels, np.int32)
        if len(p) != len(y):
            raise ValueError("eval_pred: %d pCTR values for %d labels" % (len(p), len(y)))
        if weights is not None:
            w = np.ascontiguousarray(weights, np.float32)
            if len(w) != len(p):
                raise ValueError("eval_pred: %d weights for %d rows" % (len(w), len(p)))
            loss, correct, auc = C.c_float(), C.c_double(), C.c_float()
            _chk(self.L.lctr_eval_pred_weighted(self.h, len(p), _p(p), _p(y), _p(w), C.byref(loss), C.byref(correct),
                                                C.byref(auc)))
            return loss.value, correct.value, auc.value
        loss, correct, auc = C.c_float(), C.c_int64(), C.c_float()
        _chk(self.L.lctr_eval_pred(self.h, len(p), _p(p), _p(y), C.byref(loss), C.byref(correct), C.byref(auc)))
        return loss.value, correct.value, auc.value

    def eval_weighted(self, slot):
        """(summed weighted logloss, weighted correct count, weighted AUC) of the slot's pCTR / labels under the row weights
        set with set_row_weights (lctr_eval_weighted)."""
        loss, correct, auc = C.c_float(), C.c_double(), C.c_float()
        _chk(self.L.lctr_eval_weighted(self.h, slot, C.byref(loss), C.byref(correct), C.byref(auc)))
        return loss.value, correct.value, auc.value

    def upload_pred(self, slot, pctr):
        p = np.ascontiguousarray(pctr, np.float32)
        _chk(self.L.lctr_upload_pred(self.h, slot, p.ctypes.data))

    def save_checkpoint(self, path):
        _chk(self.L.lctr_save_checkpoint(self.h, path.encode()))

    def load_checkpoint(self, path):
        _chk(self.L.lctr_load_checkpoint(self.h, path.encode()))

    def load_checkpoint_shards(self, paths):
        """The files of one save (ranks 0..n-1 of a world-n run, or one single-GPU file) into this context, whatever its
        world: this rank takes the rows it owns."""
        arr = (C.c_char_p * len(paths))(*[p.encode() for p in paths])
        _chk(self.L.lctr_load_checkpoint_shards(self.h, len(paths), arr))

    def track_changes(self, enable=True):
        """Keep (enable=True, cleared) or drop the per-row change map that incremental saves write from.  Either call
        forgets the parent: the next save or in-place load while tracking is on becomes it."""
        _chk(self.L.lctr_track_changes(self.h, 1 if enable else 0))

    def save_checkpoint_delta(self, path):
        """the rows changed since the parent save, and the small state, into `path`; returns the rows written"""
        n = C.c_uint64()
        _chk(self.L.lctr_save_checkpoint_delta(self.h, path.encode(), C.byref(n)))
        return n.value

    def load_checkpoint_chain(self, paths):
        """a full checkpoint (paths[0]) and its deltas in order, checked whole before anything is written"""
        arr = (C.c_char_p * len(paths))(*[p.encode() for p in paths])
        _chk(self.L.lctr_load_checkpoint_chain(self.h, len(paths), arr))

    def mlp_download_grad(self, layer, n_in, n_out):
        w, b = np.empty(n_in * n_out, np.float32), np.empty(n_out, np.float32)
        _chk(self.L.lctr_mlp_download_grad(self.h, layer, w.ctypes.data, b.ctypes.data))
        return w, b

    def mlp_forward(self, x):
        x = np.ascontiguousarray(x, np.float32)
        out = np.empty(x.shape[0], np.float32)
        _chk(self.L.lctr_mlp_forward(self.h, x.shape[0], x.ctypes.data, out.ctypes.data))
        return out

    def mlp_backward(self, dout, in0):
        dout = np.ascontiguousarray(dout, np.float32)
        dx = np.empty((len(dout), in0), np.float32)
        _chk(self.L.lctr_mlp_backward(self.h, len(dout), dout.ctypes.data, dx.ctypes.data))
        return dx

    def mlp_apply(self, minibatch):
        _chk(self.L.lctr_mlp_apply(self.h, minibatch))

    def mlp_set_mask(self, layer, mask):
        m = np.ascontiguousarray(mask, np.float32)
        _chk(self.L.lctr_mlp_set_mask(self.h, layer, m.ctypes.data))

    PROF_NAMES = ["fm_forward", "fm_backward_red", "apply", "ffm_fused", "fm_backward_csc", "mlp", "dist_mark", "dist_compact",
                  "dist_pull", "dist_push", "dist_barrier0", "dist_merge", "dist_barrier1", "csc_build", "fm_fused", "apply_compact",
                  "keys_translate", "text_parse"]

    def profile(self, enable=True):
        _chk(self.L.lctr_profile(self.h, 1 if enable else 0))

    def profile_read(self, reset=True):
        n = len(self.PROF_NAMES)
        ms = (C.c_double * n)()
        cnt = (C.c_int64 * n)()
        _chk(self.L.lctr_profile_read(self.h, ms, cnt, n, 1 if reset else 0))
        return {self.PROF_NAMES[i]: (ms[i], cnt[i]) for i in range(n) if cnt[i] > 0}

    def ipc_export(self):
        n = C.c_size_t()
        _chk(self.L.lctr_ipc_export(self.h, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        _chk(self.L.lctr_ipc_export(self.h, buf, n.value, C.byref(n)))
        return buf.raw

    def ipc_import(self, all_blobs, bytes_per_rank):
        buf = C.create_string_buffer(all_blobs, len(all_blobs))
        _chk(self.L.lctr_ipc_import(self.h, buf, bytes_per_rank))

    def device_bytes(self):
        a, b = C.c_uint64(), C.c_uint64()
        _chk(self.L.lctr_device_bytes(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def launch_count(self):
        return self.L.lctr_launch_count(self.h)

    def stream(self):
        return self.L.lctr_stream(self.h)
