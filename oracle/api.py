"""oracle/api.py -- TEST INFRASTRUCTURE ONLY.

ctypes bindings for oracle/liboracle.so (plain-C restatement) and, when present,
oracle/_ref/libref.so (the unmodified reference compiled in place by oracle/Makefile).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
import this module; nothing under lightctr_b200/ does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


def build(ref=True):
    """Compile the checker(s).  Building the checker is not using it."""
    subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])
    if ref and os.path.isdir("/root/reference/LightCTR"):
        subprocess.check_call(["make", "-s", "-C", HERE, "ref"])
        subprocess.check_call(["make", "-s", "-C", HERE, "refdist"])  # cluster roles; skipped by the Makefile without a libzmq


class _Data(C.Structure):
    _fields_ = [("rows", C.c_int64), ("nnz", C.c_int64), ("row_ptr", C.POINTER(C.c_int64)),
                ("fid", C.POINTER(C.c_uint64)), ("field", C.POINTER(C.c_uint64)),
                ("val", C.POINTER(C.c_float)), ("label", C.POINTER(C.c_int)), ("label_cnt", C.c_int64),
                ("feature_cnt", C.c_uint64), ("field_cnt", C.c_uint64)]


class _Mlp(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("act", C.c_int), ("dims", C.c_size_t * 17),
                ("weight", C.POINTER(C.c_float) * 16), ("bias", C.POINTER(C.c_float) * 16),
                ("mask", C.POINTER(C.c_float) * 16), ("dW", C.POINTER(C.c_float) * 16),
                ("db", C.POINTER(C.c_float) * 16), ("accum", C.POINTER(C.c_float) * 16),
                ("out_act", C.POINTER(C.c_float) * 16), ("in_delta", C.POINTER(C.c_float) * 16),
                ("input", C.POINTER(C.c_float))]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    path = os.path.join(HERE, "liboracle.so")
    if not os.path.exists(path):
        build(ref=False)
    L = C.CDLL(path)
    L.orc_srand.argtypes = [C.c_uint]
    L.orc_rand.restype = C.c_int
    L.orc_uniform.restype = C.c_double
    L.orc_gauss.restype = C.c_double
    L.orc_init_V.argtypes = [_f32p, C.c_size_t, C.c_size_t]
    L.orc_dot.argtypes = [_f32p, _f32p, C.c_size_t]
    L.orc_dot.restype = C.c_float
    L.orc_sigmoid.argtypes = [C.c_float]
    L.orc_sigmoid.restype = C.c_float
    L.orc_load.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64]
    L.orc_load.restype = C.POINTER(_Data)
    L.orc_load_test.argtypes = [C.c_char_p, C.c_uint64]
    L.orc_load_test.restype = C.POINTER(_Data)
    L.orc_free_data.argtypes = [C.POINTER(_Data)]
    L.orc_adagrad.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, C.c_size_t, C.c_float]
    L.orc_ftrl.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, _f32p, C.c_int]
    L.orc_ps_update.argtypes = [C.c_int, C.c_size_t, _f32p, _f32p, _f32p, _f32p, C.c_size_t, C.c_float, C.c_int]
    L.orc_adadelta.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, _f32p, C.c_size_t, C.c_float]
    L.orc_rmsprop.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, C.c_size_t, C.c_float, C.c_float]
    L.orc_adam.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, _f32p, C.POINTER(C.c_size_t), C.c_size_t,
                           C.c_float, C.c_float, C.c_float]
    L.orc_fm_pass.argtypes = [C.c_int64, _i64p, _u32p, _f32p, _i32p, C.c_size_t, C.c_size_t, _f32p, _f32p,
                              _f32p, _f32p, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p]
    L.orc_ffm_pass.argtypes = [C.c_int64, _i64p, _u32p, _u32p, _f32p, _i32p, C.c_size_t, C.c_size_t, C.c_size_t,
                               _f32p, _f32p, _f32p, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float),
                               C.c_void_p]
    L.orc_mlp_create.argtypes = [C.c_int, C.POINTER(C.c_size_t), C.c_int, C.c_float]
    L.orc_mlp_create.restype = C.POINTER(_Mlp)
    L.orc_mlp_free.argtypes = [C.POINTER(_Mlp)]
    L.orc_mlp_forward.argtypes = [C.POINTER(_Mlp), _f32p]
    L.orc_mlp_forward.restype = C.c_float
    L.orc_mlp_backward.argtypes = [C.POINTER(_Mlp), C.c_float]
    L.orc_mlp_apply.argtypes = [C.POINTER(_Mlp), C.c_size_t, C.c_float, C.c_float]
    L.orc_nfm_epoch.argtypes = [C.c_int64, _i64p, _u32p, _f32p, _i32p, C.c_size_t, C.c_size_t, _f32p, _f32p, _f32p,
                                _f32p, _f32p, C.POINTER(_Mlp), C.c_size_t, C.c_size_t, C.c_float, C.c_float,
                                C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_size_t)]
    L.orc_wnd_epoch.argtypes = [C.c_int64, _i64p, _u32p, _u32p, _f32p, _i32p, C.c_size_t, C.c_size_t, C.c_size_t, _f32p,
                                _f32p, _f32p, _f32p, C.POINTER(_Mlp), C.c_size_t, C.c_size_t, C.c_float, C.c_float,
                                C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_size_t)]
    L.orc_wnd_epoch_ref.argtypes = [C.c_int64, _i64p, _u32p, _u32p, _f32p, _i32p, C.c_size_t, C.c_size_t, C.c_size_t, _f32p,
                                    _f32p, _f32p, _f32p, C.POINTER(_Mlp), C.c_size_t, C.c_size_t, C.c_float, C.c_float, C.c_int,
                                    _f32p, _f32p, C.POINTER(C.c_float), C.POINTER(C.c_size_t)]
    L.orc_wire_f16.argtypes = [C.c_float]
    L.orc_wire_f16.restype = C.c_float
    L.orc_predict.argtypes = [C.c_int64, _i64p, _u32p, _u32p, _f32p, _i32p, C.c_size_t, C.c_size_t, _f32p, _f32p,
                              C.c_void_p, C.c_int, _f32p, C.POINTER(C.c_float), C.POINTER(C.c_int),
                              C.POINTER(C.c_float)]
    L.orc_auc.argtypes = [_f32p, _i32p, C.c_size_t]
    L.orc_auc.restype = C.c_float
    L.orc_murmur_u64.argtypes = [C.c_uint64]
    L.orc_murmur_u64.restype = C.c_uint32
    L.orc_dht_node.argtypes = [C.c_uint64, C.c_uint32]
    L.orc_dht_node.restype = C.c_uint32
    L.orc_ring_segments.argtypes = [C.c_size_t, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.orc_ring_allreduce.argtypes = [C.POINTER(C.POINTER(C.c_float)), C.c_size_t, C.c_size_t, C.c_int]
    _lib = L
    return L


# --------------------------------------------------------------------------------------------------
# numpy-level helpers around the C oracle
# --------------------------------------------------------------------------------------------------
class Dataset:
    """CSR view of FM_Algo_Abst::dataSet/label (fm_algo_abst.h:156,170)."""

    def __init__(self, row_ptr, fid, field, val, label, feature_cnt, field_cnt):
        self.row_ptr = np.ascontiguousarray(row_ptr, np.int64)
        self.fid = np.ascontiguousarray(fid, np.uint32)
        self.field = np.ascontiguousarray(field, np.uint32)
        self.val = np.ascontiguousarray(val, np.float32)
        self.label = np.ascontiguousarray(label, np.int32)
        self.feature_cnt = int(feature_cnt)
        self.field_cnt = int(field_cnt)

    @property
    def rows(self):
        return len(self.row_ptr) - 1

    @property
    def nnz(self):
        return len(self.fid)


def _from_cdata(dp):
    d = dp.contents
    rows, nnz = d.rows, d.nnz
    ds = Dataset(np.ctypeslib.as_array(d.row_ptr, (rows + 1,)).copy(),
                 np.ctypeslib.as_array(d.fid, (max(nnz, 1),))[:nnz].astype(np.uint32),
                 np.ctypeslib.as_array(d.field, (max(nnz, 1),))[:nnz].astype(np.uint32),
                 np.ctypeslib.as_array(d.val, (max(nnz, 1),))[:nnz].copy(),
                 np.ctypeslib.as_array(d.label, (max(d.label_cnt, 1),))[:d.label_cnt].copy(),
                 d.feature_cnt, d.field_cnt)
    lib().orc_free_data(dp)
    return ds


def load(path, field_cnt=0, feature_cnt=0):
    dp = lib().orc_load(path.encode(), field_cnt, feature_cnt)
    if not dp:
        raise IOError(path)
    return _from_cdata(dp)


def load_test(path, train_feature_cnt):
    dp = lib().orc_load_test(path.encode(), train_feature_cnt)
    if not dp:
        raise IOError(path)
    return _from_cdata(dp)


def init_params(seed, F, k, field_cnt=0):
    """srand(seed); W=0; V=GaussRand()/sqrt(k)  (fm_algo_abst.h:53-68)."""
    L = lib()
    L.orc_srand(seed)
    L.orc_gauss_reset()
    n = F * k * (field_cnt if field_cnt > 0 else 1)
    V = np.empty(n, np.float32)
    L.orc_init_V(V, n, k)
    return np.zeros(F, np.float32), V


class FMOracle:
    """Train_FM_Algo restated (train/train_fm_algo.cpp): one call to epoch() == one reference epoch."""

    def __init__(self, ds, k, W, V, lr=0.05, l2=0.001):
        self.ds, self.k, self.lr, self.l2 = ds, k, np.float32(lr), np.float32(l2)
        self.W, self.V = W.copy(), V.copy()
        F = ds.feature_cnt
        self.update_g = np.zeros(F * (k + 1), np.float32)
        self.accum = np.zeros(F * (k + 1), np.float32)
        self.sumVX = np.zeros(ds.rows * k, np.float32)
        self.pred = np.zeros(ds.rows, np.float32)

    def forward_backward(self):
        ds, k, F = self.ds, self.k, self.ds.feature_cnt
        self.update_g[:] = 0
        self.sumVX[:] = 0  # flash() train_fm_algo.cpp:28-33
        loss, acc = C.c_float(0), C.c_float(0)
        lib().orc_fm_pass(ds.rows, ds.row_ptr, ds.fid, ds.val, ds.label, F, k, self.W, self.V, self.sumVX,
                          self.update_g, self.l2, C.byref(loss), C.byref(acc), self.pred.ctypes.data)
        return loss.value, float(np.float32(acc.value) / np.float32(ds.rows))

    def apply(self):
        F, k = self.ds.feature_cnt, self.k
        L = lib()
        # ApplyGrad train_fm_algo.cpp:120-126 ; minibatch_size = dataRow_cnt (:38).  `opt` switches the type of the
        # trainer's `updater` member (adagrad is the shipped one); W call first, then V call, as in the reference
        opt = getattr(self, "opt", "adagrad")
        B = self.ds.rows
        if opt in ("ftrl", "adam", "adadelta", "ps_dcasgd", "ps_dcasgda") and not hasattr(self, "s2"):
            self.s2 = np.zeros(F * (k + 1), np.float32)
            self.iter = C.c_size_t(0)
        if opt in ("ps_adagrad", "ps_dcasgda") and not getattr(self, "_ps_init", False):
            self.accum[:] = np.float32(1e-7)  # data_accum = TValue(1e-7), paramserver.h:323
            self._ps_init = True
        if not hasattr(self, "s2"):
            self.s2 = np.zeros(1, np.float32)
        for (w, lo, hi) in ((self.W, 0, F), (self.V, F, F * (k + 1))):
            g, a = self.update_g[lo:hi], self.accum[lo:hi]
            if opt == "adagrad":
                L.orc_adagrad(hi - lo, w, g, a, B, self.lr)
            elif opt == "rmsprop":
                L.orc_rmsprop(hi - lo, w, g, a, B, self.lr, np.float32(getattr(self, "ema", 0.99)))
            elif opt == "adadelta":
                L.orc_adadelta(hi - lo, w, g, a, self.s2[lo:hi], B, np.float32(getattr(self, "beta1", 0.8)))
            elif opt == "ftrl":
                L.orc_ftrl(hi - lo, w, g, a, self.s2[lo:hi], 1)
            elif opt == "adam":
                L.orc_adam(hi - lo, w, g, a, self.s2[lo:hi], C.byref(self.iter), B, self.lr,
                           np.float32(getattr(self, "beta1", 0.8)), np.float32(getattr(self, "beta2", 0.999)))
            elif opt.startswith("ps_"):
                # the PS only touches the keys a worker pushed (paramserver.h:214-216): the batch's features, and of
                # those only the coordinates whose gradient is nonzero -- the worker never pushes a zero
                # (Value::checkPreferredValue, push.h:62-65), so a zero leaves DCASGD's shadow and DCASGDA's decay alone
                kind = {"ps_sgd": 0, "ps_adagrad": 1, "ps_dcasgd": 2, "ps_dcasgda": 3}[opt]
                keys = np.unique(self.ds.fid).astype(np.int64)
                idx = keys if lo == 0 else (keys[:, None] * k + np.arange(k)[None, :]).ravel()
                idx = idx[g[idx] != 0]
                ww, gg, aa = w[idx].copy(), g[idx].copy(), a[idx].copy()
                sh = self.s2[lo:hi][idx].copy() if kind >= 2 else np.zeros(1, np.float32)
                L.orc_ps_update(kind, len(idx), ww, gg, aa, sh, B, self.lr, 0)
                w[idx], a[idx] = ww, aa
                if kind >= 2:
                    self.s2[lo:hi][idx] = sh
            else:
                raise ValueError(opt)

    def epoch(self):
        r = self.forward_backward()
        self.apply()
        return r


class FFMOracle:
    """Train_FFM_Algo restated (train/train_ffm_algo.cpp).  optimizer in {adagrad, ftrl, adam, rmsprop, adadelta}."""

    def __init__(self, ds, k, W, V, lr=0.05, l2=0.001, optimizer="adagrad", beta1=0.8, beta2=0.999, ema=0.99):
        self.ema = np.float32(ema)
        self.ds, self.k, self.lr, self.l2 = ds, k, np.float32(lr), np.float32(l2)
        self.W, self.V = W.copy(), V.copy()
        self.opt = optimizer
        F, Fc = ds.feature_cnt, ds.field_cnt
        n = F * Fc * k + F
        self.update_g = np.zeros(n, np.float32)
        self.s1 = np.zeros(n, np.float32)  # adagrad accum | ftrl z | adam m
        self.s2 = np.zeros(n, np.float32)  # ftrl n | adam v
        self.iter = C.c_size_t(0)
        self.beta1, self.beta2 = np.float32(beta1), np.float32(beta2)
        self.pred = np.zeros(ds.rows, np.float32)

    def forward_backward(self):
        ds = self.ds
        loss, acc = C.c_float(0), C.c_float(0)
        lib().orc_ffm_pass(ds.rows, ds.row_ptr, ds.fid, ds.field, ds.val, ds.label, ds.feature_cnt, ds.field_cnt,
                           self.k, self.W, self.V, self.update_g, self.l2, C.byref(loss), C.byref(acc),
                           self.pred.ctypes.data)
        return loss.value, float(np.float32(acc.value) / np.float32(ds.rows))

    def apply(self):
        F = self.ds.feature_cnt
        L = lib()
        B = self.ds.rows
        for (w, lo, hi) in ((self.W, 0, F), (self.V, F, len(self.update_g))):
            g, a, b = self.update_g[lo:hi], self.s1[lo:hi], self.s2[lo:hi]
            if self.opt == "adagrad":
                L.orc_adagrad(hi - lo, w, g, a, B, self.lr)
            elif self.opt == "rmsprop":
                L.orc_rmsprop(hi - lo, w, g, a, B, self.lr, self.ema)
            elif self.opt == "adadelta":
                L.orc_adadelta(hi - lo, w, g, a, b, B, self.beta1)
            elif self.opt == "ftrl":
                L.orc_ftrl(hi - lo, w, g, a, b, 1)
            elif self.opt == "adam":
                # the reference increments iter per update() call (momentumUpdater.h:191): W call, then V call
                L.orc_adam(hi - lo, w, g, a, b, C.byref(self.iter), B, self.lr, self.beta1, self.beta2)
            else:
                raise ValueError(self.opt)

    def epoch(self):
        r = self.forward_backward()
        self.apply()
        return r


class Mlp:
    def __init__(self, dims, act=0, sparse_rate=0.8):
        arr = (C.c_size_t * len(dims))(*dims)
        self.dims = list(dims)
        self.p = lib().orc_mlp_create(len(dims) - 1, arr, act, sparse_rate)

    def arrays(self, name, l):
        m = self.p.contents
        i, o = self.dims[l], self.dims[l + 1]
        n = {"weight": i * o, "dW": i * o, "bias": o, "db": o, "mask": o, "accum": o * (i + 1), "out_act": o,
             "in_delta": i}[name]
        return np.ctypeslib.as_array(getattr(m, name)[l], (n,))

    def __del__(self):
        try:
            lib().orc_mlp_free(self.p)
        except Exception:
            pass


class NFMOracle:
    """Train_NFM_Algo restated (train/train_nfm_algo.cpp) with an arbitrary FC chain dims=[k, H.., 1].

    RNG order == reference ctor: V init (fm_algo_abst.h:62-65) then FC layers input->output
    (fullyconnLayer.h:48-54); pass seed to reproduce it, or W/V explicitly."""

    def __init__(self, ds, k, hidden, seed=None, W=None, V=None, lr=0.05, l2=0.001, batch_size=50,
                 minibatch=50, sparse_rate=0.8, act=0):
        self.ds, self.k = ds, k
        F = ds.feature_cnt
        if seed is not None:
            self.W, self.V = init_params(seed, F, k)
        else:
            self.W, self.V = W.copy(), V.copy()
        hidden = list(hidden) if isinstance(hidden, (list, tuple)) else [hidden]
        self.mlp = Mlp([k] + hidden + [1], act, sparse_rate)
        self.update_g = np.zeros(F * (k + 1), np.float32)
        self.accum = np.zeros(F * (k + 1), np.float32)
        self.sumVX = np.zeros(ds.rows * k, np.float32)
        self.lr, self.l2, self.bs, self.mb, self.sr = lr, l2, batch_size, minibatch, sparse_rate

    def epoch(self):
        ds = self.ds
        loss, acc = C.c_float(0), C.c_size_t(0)
        lib().orc_nfm_epoch(ds.rows, ds.row_ptr, ds.fid, ds.val, ds.label, ds.feature_cnt, self.k, self.W, self.V,
                            self.sumVX, self.update_g, self.accum, self.mlp.p, self.bs, self.mb, self.lr, self.l2,
                            self.sr, C.byref(loss), C.byref(acc))
        return loss.value, acc.value / ds.rows


class WNDOracle:
    """Wide&Deep with per-field concat input (Distributed_Algo_Abst::batchGradCompute).  dims = [Fc*d, H.., 1].
    schedule="sync" (default): one synchronous process, gradients applied once per minibatch -- what the CUDA path implements.
    schedule="reference": the cluster's own schedule (binary16 wire, per-sample tensor SGD on the server, wide weights pulled
    and pushed once per minibatch; optimizer is the server's SGD, l2 = 0) -- PINNED against a real Master + ParamServer +
    worker run, tests/golden/wnd_ref_curve.json / tests/test_oracle_wnd_pin_cpu.py."""

    def __init__(self, ds, d, hidden, W, E, lr=0.05, l2=0.001, batch_size=50, minibatch=50, sparse_rate=0.8, act=0,
                 optimizer="adagrad", schedule="sync"):
        self.ds, self.d = ds, d
        self.schedule = schedule
        self.ps_rule = 1 if optimizer == "ps_sgd" else 0
        self.ps_kind = {"ps_sgd": 0, "ps_adagrad": 1, "ps_dcasgd": 2, "ps_dcasgda": 3}.get(optimizer, 0)
        if schedule == "reference":  # the server's per-key state: data_accum starts at 1e-7, shadow copies at 0 (paramserver.h:318-327)
            self.ps_accum = np.full(ds.feature_cnt, 1e-7, np.float32)
            self.ps_shadow = np.zeros(ds.feature_cnt, np.float32)
        F, Fc = ds.feature_cnt, ds.field_cnt
        self.W, self.E = W.copy(), E.copy()
        hidden = list(hidden) if isinstance(hidden, (list, tuple)) else [hidden]
        self.mlp = Mlp([Fc * d] + hidden + [1], act, sparse_rate)
        self.update_g = np.zeros(F * (d + 1), np.float32)
        self.accum = np.zeros(F * (d + 1), np.float32)
        self.lr, self.l2, self.bs, self.mb, self.sr = lr, l2, batch_size, minibatch, sparse_rate

    def epoch(self):
        ds = self.ds
        loss, acc = C.c_float(0), C.c_size_t(0)
        if self.schedule == "reference":
            pulled = np.zeros(ds.feature_cnt, np.float32)
            lib().orc_wnd_epoch_ref(ds.rows, ds.row_ptr, ds.fid, ds.field, ds.val, ds.label, ds.feature_cnt, ds.field_cnt, self.d,
                                    self.W, self.E, self.update_g[:ds.feature_cnt], pulled, self.mlp.p, self.bs, self.mb, self.lr,
                                    self.sr, self.ps_kind, self.ps_accum, self.ps_shadow, C.byref(loss), C.byref(acc))
            return loss.value, acc.value / ds.rows
        lib().orc_set_wnd_ps_rule(self.ps_rule)
        lib().orc_wnd_epoch(ds.rows, ds.row_ptr, ds.fid, ds.field, ds.val, ds.label, ds.feature_cnt, ds.field_cnt, self.d,
                            self.W, self.E, self.update_g, self.accum, self.mlp.p, self.bs, self.mb, self.lr, self.l2,
                            self.sr, C.byref(loss), C.byref(acc))
        return loss.value, acc.value / ds.rows


def predict(test, Fc, k, W, V, train_sumVX, is_ffm):
    pctr = np.zeros(test.rows, np.float32)
    loss, correct, auc = C.c_float(0), C.c_int(0), C.c_float(0)
    lib().orc_predict(test.rows, test.row_ptr, test.fid, test.field, test.val, test.label, Fc, k, W, V,
                      None if train_sumVX is None else train_sumVX.ctypes.data, int(is_ffm), pctr,
                      C.byref(loss), C.byref(correct), C.byref(auc))
    return pctr, loss.value, correct.value, auc.value


# --------------------------------------------------------------------------------------------------
# the compiled reference (oracle/_ref/libref.so)
# --------------------------------------------------------------------------------------------------
_ref = None


def ref_available():
    return os.path.exists(os.path.join(HERE, "_ref", "libref.so"))


def ref():
    global _ref
    if _ref is not None:
        return _ref
    R = C.CDLL(os.path.join(HERE, "_ref", "libref.so"))
    R.ref_set_hyper.argtypes = [C.c_size_t] + [C.c_float] * 7
    for n in ("ref_fm_create", "ref_ffm_create", "ref_nfm_create"):
        getattr(R, n).restype = C.c_void_p
    R.ref_fm_create.argtypes = [C.c_char_p, C.c_int, C.c_uint, C.c_int]
    R.ref_ffm_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_uint, C.c_int]
    R.ref_nfm_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_uint]
    R.ref_destroy.argtypes = [C.c_void_p]
    R.ref_dims.argtypes = [C.c_void_p] + [C.POINTER(C.c_size_t)] * 5
    R.ref_get_data.argtypes = [C.c_void_p, _i64p, _u64p, _u64p, _f32p, _i32p]
    R.ref_get_params.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    R.ref_set_params.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    R.ref_train_epoch.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    R.ref_nfm_get_fc.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    R.ref_time_train.argtypes = [C.c_void_p, C.c_int]
    R.ref_time_train.restype = C.c_double
    R.ref_predict.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    R.ref_adagrad_update.argtypes = [C.c_size_t, C.c_size_t, C.c_float, _f32p, _f32p, _f32p]
    R.ref_ftrl_update.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, _f32p]
    R.ref_adadelta_update.argtypes = [C.c_size_t, C.c_size_t, C.c_float, _f32p, _f32p, _f32p, _f32p]
    R.ref_rmsprop_update.argtypes = [C.c_size_t, C.c_size_t, C.c_float, C.c_float, _f32p, _f32p, _f32p]
    R.ref_adam_update.argtypes = [C.c_size_t, C.c_size_t, C.c_float, C.c_float, C.c_float, C.c_size_t, _f32p, _f32p,
                                  _f32p, _f32p]
    R.ref_sigmoid.argtypes = [C.c_float]
    R.ref_sigmoid.restype = C.c_float
    R.ref_dot.argtypes = [_f32p, _f32p, C.c_size_t]
    R.ref_dot.restype = C.c_float
    R.ref_gauss_fill.argtypes = [C.c_uint, C.c_size_t, C.c_size_t, _f32p]
    R.ref_hw_threads.restype = C.c_uint
    _ref = R
    return R


DEFAULT_HYPER = dict(minibatch=50, lr=0.05, ema=0.99, sparse_rate=0.8, l2=0.001, l1=1e-5, momentum=0.8, adam2=0.999)


class RefTrainer:
    """Handle on a reference trainer object (Train_FM_Algo / Train_FFM_Algo / Train_NFM_Algo)."""

    def __init__(self, kind, path, k, seed=1, proc_cnt=1, field_cnt=0, hidden=32, **hyper):
        R = ref()
        hp = dict(DEFAULT_HYPER)
        hp.update(hyper)
        R.ref_set_hyper(hp["minibatch"], hp["lr"], hp["ema"], hp["sparse_rate"], hp["l2"], hp["l1"], hp["momentum"],
                        hp["adam2"])
        self.kind = kind
        if kind == "fm":
            self.h = R.ref_fm_create(path.encode(), k, seed, proc_cnt)
        elif kind == "ffm":
            self.h = R.ref_ffm_create(path.encode(), k, field_cnt, seed, proc_cnt)
        elif kind == "nfm":
            self.h = R.ref_nfm_create(path.encode(), k, hidden, seed)
        else:
            raise ValueError(kind)
        d = [C.c_size_t() for _ in range(5)]
        R.ref_dims(self.h, *[C.byref(x) for x in d])
        self.rows, self.nnz, self.feature_cnt, self.field_cnt, self.factor_cnt = [x.value for x in d]

    def data(self):
        rp = np.zeros(self.rows + 1, np.int64)
        fid = np.zeros(self.nnz, np.uint64)
        fld = np.zeros(self.nnz, np.uint64)
        val = np.zeros(self.nnz, np.float32)
        lab = np.zeros(self.rows, np.int32)
        ref().ref_get_data(self.h, rp, fid, fld, val, lab)
        return Dataset(rp, fid, fld, val, lab, self.feature_cnt, self.field_cnt)

    def params(self):
        F, k = self.feature_cnt, self.factor_cnt
        nv = F * k * (self.field_cnt if self.field_cnt > 0 else 1)
        W = np.zeros(F, np.float32)
        V = np.zeros(nv, np.float32)
        S = np.zeros(self.rows * k, np.float32)
        ref().ref_get_params(self.h, W.ctypes.data, V.ctypes.data, S.ctypes.data if self.kind != "ffm" else None)
        return W, V, S

    def set_params(self, W, V):
        ref().ref_set_params(self.h, W.ctypes.data, V.ctypes.data)

    def epoch(self):
        loss, acc = C.c_float(), C.c_float()
        ref().ref_train_epoch(self.h, C.byref(loss), C.byref(acc))
        return loss.value, acc.value

    def fc(self, layer, n_in, n_out):
        w = np.zeros(n_in * n_out, np.float32)
        b = np.zeros(n_out, np.float32)
        m = np.zeros(n_out, np.float32)
        ref().ref_nfm_get_fc(self.h, layer, w.ctypes.data, b.ctypes.data, m.ctypes.data)
        return w, b, m

    def time_train(self, epochs):
        return ref().ref_time_train(self.h, epochs)

    def predict(self, test_path, save_path=None):
        buf = C.create_string_buffer(4096)
        ref().ref_predict(self.h, test_path.encode(), save_path.encode() if save_path else None, buf, 4096)
        return buf.value.decode()

    def close(self):
        if self.h:
            ref().ref_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
