"""ctypes binding of include/difacto_b200.h (no CPU fallback: raises if the library is absent)."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DFB_LIB") or os.path.join(HERE, "lib", "libdifacto_b200.so")   # DFB_LIB: a tuning build

DFB_OK, DFB_ERR_INVALID, DFB_ERR_CUDA, DFB_ERR_CAPACITY, DFB_ERR_PARAM = 0, -1, -2, -3, -4


class DfbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"difacto_b200 error {code}: {msg}")
        self.code = code


class Progress(C.Structure):
    _fields_ = [("loss", C.c_float), ("penalty", C.c_float), ("auc", C.c_float), ("nnz_w", C.c_float),
                ("nrows", C.c_float), ("new_keys", C.c_uint64), ("new_vrows", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


EXPORTS = [
    "dfb_create", "dfb_destroy", "dfb_last_error", "dfb_num_unknown_kwargs", "dfb_unknown_kwarg",
    "dfb_launch_count", "dfb_table_stats", "dfb_host_alloc", "dfb_host_free", "dfb_push_feacnt",
    "dfb_pull", "dfb_push_grad", "dfb_predict", "dfb_calc_grad", "dfb_evaluate", "dfb_auc",
    "dfb_train_step", "dfb_train_step_dev", "dfb_sync", "dfb_read_progress", "dfb_train_step_async",
    "dfb_read_entries", "dfb_rng_state", "dfb_key_owner", "dfb_shard_bounds", "dfb_row_stride",
    "dfb_dev_feacnt", "dfb_dev_pull_rows", "dfb_dev_fm_step", "dfb_dev_push_rows", "dfb_stream",
    "dfb_wait_step", "dfb_profile", "dfb_profile_read",
    "dfb_peer_alloc", "dfb_peer_open", "dfb_peer_close", "dfb_peer_free", "dfb_dev_pull_rows_peer",
    "dfb_dev_fm_step_peer", "dfb_localize", "dfb_train_step_raw", "dfb_train_step_raw_async",
    "dfb_train_step_raw_dev", "dfb_prefetch_raw", "dfb_snapshot_size", "dfb_snapshot", "dfb_restore",
    "dfb_snapshot_write", "dfb_restore_read", "dfb_snapshot_begin", "dfb_frozen_write", "dfb_frozen_error",
    "dfb_frozen_release", "dfb_id_range_get", "dfb_id_range_set", "dfb_prune", "dfb_prune_rare",
    "dfb_shard_init", "dfb_shard_export", "dfb_shard_connect", "dfb_shard_step_dev", "dfb_shard_step_async",
    "dfb_shard_info", "dfb_shard_begin_async", "dfb_shard_begin_dev", "dfb_shard_phase", "dfb_time_mark", "dfb_time_elapsed_ms",
    "dfb_predict_raw_async", "dfb_predict_raw_dev", "dfb_shard_predict_async", "dfb_shard_begin_predict_async",
    "dfb_row_bytes", "dfb_growth_stats",
]

_LIB = None

# dfb_write_fn / dfb_read_fn of the streamed checkpoint
WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)
READ_FN = C.CFUNCTYPE(C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t)
READ_ERROR = 2 ** 64 - 1     # (size_t)-1


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
        L.dfb_create.argtypes = [vp, vp, C.c_int, C.POINTER(vp)]
        L.dfb_destroy.argtypes = [vp]
        L.dfb_last_error.restype = C.c_char_p
        L.dfb_last_error.argtypes = [vp]
        L.dfb_num_unknown_kwargs.argtypes = [vp]
        L.dfb_unknown_kwarg.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
        L.dfb_launch_count.restype = u64
        L.dfb_launch_count.argtypes = [vp]
        L.dfb_table_stats.argtypes = [vp] + [C.POINTER(u64)] * 4
        L.dfb_row_bytes.argtypes = [vp] + [C.POINTER(u64)] * 2
        L.dfb_growth_stats.argtypes = [vp] + [C.POINTER(u64)] * 2
        L.dfb_host_alloc.argtypes = [C.POINTER(vp), sz]
        L.dfb_host_free.argtypes = [vp]
        L.dfb_push_feacnt.argtypes = [vp, vp, sz, vp]
        L.dfb_pull.argtypes = [vp, vp, sz, vp, sz, vp, C.POINTER(sz), C.POINTER(sz)]
        L.dfb_push_grad.argtypes = [vp, vp, sz, vp, sz, vp, sz]
        L.dfb_predict.argtypes = [vp, sz, vp, vp, vp, vp, sz, vp, vp, sz, vp]
        L.dfb_calc_grad.argtypes = [vp, sz, vp, vp, vp, vp, vp, sz, vp, vp, sz, vp, vp]
        L.dfb_evaluate.argtypes = [vp, vp, vp, sz, C.POINTER(C.c_float)]
        L.dfb_auc.argtypes = [vp, vp, vp, sz, C.POINTER(C.c_float)]
        L.dfb_train_step.argtypes = [vp, sz, vp, vp, vp, vp, vp, sz, vp, C.c_int, C.POINTER(Progress), vp]
        L.dfb_train_step_dev.argtypes = [vp, sz, sz, vp, vp, vp, vp, vp, sz, vp, C.c_int]
        L.dfb_train_step_async.argtypes = [vp, sz, vp, vp, vp, vp, vp, sz, vp, C.c_int]
        L.dfb_sync.argtypes = [vp]
        L.dfb_read_progress.argtypes = [vp, C.POINTER(Progress)]
        L.dfb_read_entries.argtypes = [vp, vp, sz, vp, vp, vp, vp]
        L.dfb_rng_state.argtypes = [vp, C.POINTER(C.c_uint32)]
        L.dfb_key_owner.restype = C.c_uint32
        L.dfb_key_owner.argtypes = [u64, C.c_uint32]
        L.dfb_shard_bounds.argtypes = [vp, sz, C.c_uint32, vp]
        L.dfb_row_stride.argtypes = [vp]
        L.dfb_dev_feacnt.argtypes = [vp, vp, sz, vp]
        L.dfb_dev_pull_rows.argtypes = [vp, vp, sz, vp, vp, vp]
        L.dfb_dev_fm_step.argtypes = [vp, sz, sz, vp, vp, vp, vp, sz, vp, vp, vp, C.c_int, vp, vp]
        L.dfb_dev_push_rows.argtypes = [vp, vp, sz, vp, vp, vp]
        L.dfb_wait_step.argtypes = [vp, C.POINTER(Progress)]
        L.dfb_profile.argtypes = [vp, C.c_int]
        L.dfb_profile_read.argtypes = [vp, vp, vp]
        L.dfb_peer_alloc.argtypes = [vp, sz, C.POINTER(vp), vp]
        L.dfb_peer_open.argtypes = [vp, vp, C.POINTER(vp)]
        L.dfb_peer_close.argtypes = [vp, vp]
        L.dfb_peer_free.argtypes = [vp, vp]
        L.dfb_dev_pull_rows_peer.argtypes = [vp, vp, sz, vp, vp, vp, vp]
        L.dfb_dev_fm_step_peer.argtypes = [vp, sz, sz, vp, vp, vp, vp, sz, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int]
        L.dfb_localize.argtypes = [vp, sz, vp, vp, u64, vp, vp, vp, C.POINTER(sz)]
        L.dfb_train_step_raw.argtypes = [vp, sz, vp, vp, vp, vp, C.c_int, C.c_int, C.POINTER(Progress), vp]
        L.dfb_train_step_raw_async.argtypes = [vp, sz, vp, vp, vp, vp, C.c_int, C.c_int]
        L.dfb_prefetch_raw.argtypes = [vp, sz, vp, vp, vp, vp]
        L.dfb_train_step_raw_dev.argtypes = [vp, sz, sz, vp, vp, vp, vp, C.c_int, C.c_int]
        L.dfb_snapshot_size.argtypes = [vp, C.c_int, C.POINTER(sz)]
        L.dfb_snapshot.argtypes = [vp, C.c_int, vp, sz]
        L.dfb_restore.argtypes = [vp, vp, sz, C.POINTER(C.c_int)]
        L.dfb_snapshot_write.argtypes = [vp, C.c_int, sz, WRITE_FN, vp]
        L.dfb_restore_read.argtypes = [vp, READ_FN, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, sz,
                                       C.POINTER(C.c_int)]
        L.dfb_snapshot_begin.argtypes = [vp, C.c_int, C.POINTER(vp)]
        L.dfb_frozen_write.argtypes = [vp, sz, WRITE_FN, vp]
        L.dfb_frozen_error.restype = C.c_char_p
        L.dfb_frozen_error.argtypes = [vp]
        L.dfb_frozen_release.argtypes = [vp]
        L.dfb_id_range_get.argtypes = [vp, C.POINTER(C.c_int)]
        L.dfb_id_range_set.argtypes = [vp, C.c_int]
        L.dfb_prune.argtypes = [vp, C.c_float, C.POINTER(u64)]
        L.dfb_prune_rare.argtypes = [vp, C.c_float, C.POINTER(u64), C.POINTER(u64)]
        L.dfb_shard_init.argtypes = [vp, C.c_int, C.c_int, sz, sz, sz, sz, C.POINTER(sz)]
        L.dfb_shard_export.argtypes = [vp, C.POINTER(vp), vp]
        L.dfb_shard_connect.argtypes = [vp, vp]
        L.dfb_shard_step_dev.argtypes = [vp, sz, sz, vp, vp, vp, vp, C.c_int, C.c_int]
        L.dfb_shard_step_async.argtypes = [vp, sz, vp, vp, vp, vp, C.c_int, C.c_int]
        L.dfb_time_mark.argtypes = [vp, C.c_int]
        L.dfb_time_elapsed_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.dfb_shard_begin_async.argtypes = [vp, sz, vp, vp, vp, vp, C.c_int, C.c_int]
        L.dfb_shard_begin_dev.argtypes = [vp, sz, sz, vp, vp, vp, vp, C.c_int, C.c_int]
        L.dfb_shard_phase.argtypes = [vp, C.c_int]
        L.dfb_predict_raw_async.argtypes = [vp, sz, vp, vp, vp, vp, vp]
        L.dfb_predict_raw_dev.argtypes = [vp, sz, sz, vp, vp, vp, vp, vp]
        L.dfb_shard_predict_async.argtypes = [vp, sz, vp, vp, vp, vp, vp]
        L.dfb_shard_begin_predict_async.argtypes = [vp, sz, vp, vp, vp, vp, vp]
        L.dfb_shard_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(sz), C.POINTER(sz),
                                     C.POINTER(u64)]
        L.dfb_stream.restype = vp
        L.dfb_stream.argtypes = [vp]
        _LIB = L
    return _LIB


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if isinstance(a, int):
        return C.c_void_p(a)
    return C.c_void_p(a.data_ptr())   # torch tensor


def _arr(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


def _write_cb(fileobj, failed):
    def write(_ctx, buf, n):
        try:
            fileobj.write(C.string_at(buf, n))
            return 0
        except Exception as e:     # reported after the C call returns
            failed.append(e)
            return 1
    return WRITE_FN(write)


class Frozen:
    """a snapshot frozen on the device by Engine.snapshot_begin (wraps a dfb_frozen).  write_to may run on another
    thread while the engine trains; release frees the copy (closing the engine frees one not released, after which
    write_to refuses and release does nothing)."""

    def __init__(self, engine, f):
        self.engine, self.f, self.L = engine, f, engine.L

    def write_to(self, fileobj, chunk_bytes=0):
        if not self.f:
            raise DfbError(DFB_ERR_INVALID, "the frozen snapshot was released")
        failed = []
        cb = _write_cb(fileobj, failed)
        rc = self.L.dfb_frozen_write(self.f, int(chunk_bytes), cb, None)
        if rc != 0:
            err = DfbError(rc, self.L.dfb_frozen_error(self.f).decode())
            if failed:
                raise err from failed[0]
            raise err

    def release(self):
        if self.f:
            self.L.dfb_frozen_release(self.f)
            self.f = None


def key_owner(key, S):
    return lib().dfb_key_owner(int(key), int(S))


def shard_bounds(sorted_keys, S):
    keys = _arr(sorted_keys, np.uint64)
    out = np.zeros(S + 1, dtype=np.uint64)
    rc = lib().dfb_shard_bounds(_p(keys), len(keys), S, _p(out))
    if rc != 0:
        raise DfbError(rc, "dfb_shard_bounds")
    return out.astype(np.int64)


class Engine:
    """One shard of the model on one GPU (wraps a dfb_handle).

    The keyword arguments are dfb_create's keys (include/difacto_b200.h).  table_capacity / V_capacity are the initial
    capacities; with table_capacity_max / V_capacity_max above them the table and the V-row pool grow on demand, and
    table_stats() reports the current capacities; shard_growth=1 lets such an engine be a rank of the fused sharded
    store, whose owners then grow by the keys they receive.  score_only=True (optionally V_storage="bf16") makes a scoring-only
    engine: restore and predict_raw* only, V rows without their AdaGrad halves; what it refuses raises DfbError.  It may
    also be a rank of a fused sharded store of two or more ranks (shard_init), which then runs shard_predict_async /
    shard_begin_predict_async only."""

    def __init__(self, **kwargs):
        L = lib()
        ks = [str(k).encode() for k in kwargs]
        vs = [str(int(v) if isinstance(v, bool) else v).encode() for v in kwargs.values()]
        n = len(ks)
        ka = (C.c_char_p * n)(*ks)
        va = (C.c_char_p * n)(*vs)
        h = C.c_void_p()
        rc = L.dfb_create(ka, va, n, C.byref(h))
        if rc != 0:
            raise DfbError(rc, L.dfb_last_error(None).decode())
        self.h = h
        self.V_dim = int(kwargs["V_dim"])
        self.L = L

    def close(self):
        if getattr(self, "h", None):
            for f in getattr(self, "_frozen", []):
                f.f = None           # dfb_destroy releases a frozen snapshot left behind
            self.L.dfb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise DfbError(rc, self.L.dfb_last_error(self.h).decode())

    # ---- misc ----
    def unknown_kwargs(self):
        out = []
        for i in range(self.L.dfb_num_unknown_kwargs(self.h)):
            k, v = C.c_char_p(), C.c_char_p()
            self.L.dfb_unknown_kwarg(self.h, i, C.byref(k), C.byref(v))
            out.append((k.value.decode(), v.value.decode()))
        return out

    def launch_count(self):
        return int(self.L.dfb_launch_count(self.h))

    def table_stats(self):
        a, b, c, d = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        self._ck(self.L.dfb_table_stats(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return dict(n_keys=a.value, n_vrows=b.value, capacity=c.value, v_capacity=d.value)

    def growth_stats(self):
        """(calls that grew the table or the V-row pool, sharded growth decisions that waited for the device)"""
        a, b = C.c_uint64(), C.c_uint64()
        self._ck(self.L.dfb_growth_stats(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def row_bytes(self):
        """(bytes one V row takes in the row pool, n_vrows times that)"""
        a, b = C.c_uint64(), C.c_uint64()
        self._ck(self.L.dfb_row_bytes(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def rng_state(self):
        s = C.c_uint32()
        self._ck(self.L.dfb_rng_state(self.h, C.byref(s)))
        return s.value

    def row_stride(self):
        return self.L.dfb_row_stride(self.h)

    def stream(self):
        return self.L.dfb_stream(self.h)

    # ---- (A) Store / Updater / Loss mirror ----
    def push_feacnt(self, keys, cnt):
        keys, cnt = _arr(keys, np.uint64), _arr(cnt, np.float32)
        self._ck(self.L.dfb_push_feacnt(self.h, _p(keys), len(keys), _p(cnt)))

    def pull(self, keys):
        keys = _arr(keys, np.uint64)
        n = len(keys)
        vals = np.zeros(max(n * (1 + self.V_dim), 1), np.float32)
        lens = np.zeros(max(n, 1), np.int32)
        nv, nl = C.c_size_t(), C.c_size_t()
        self._ck(self.L.dfb_pull(self.h, _p(keys), n, _p(vals), len(vals), _p(lens), C.byref(nv), C.byref(nl)))
        return vals[:nv.value].copy(), lens[:nl.value].copy()

    def push_grad(self, keys, grads, lens):
        keys, grads = _arr(keys, np.uint64), _arr(grads, np.float32)
        lens = _arr(lens, np.int32)
        nl = 0 if lens is None else len(lens)
        self._ck(self.L.dfb_push_grad(self.h, _p(keys), len(keys), _p(grads), len(grads),
                                      _p(lens) if nl else None, nl))

    def predict(self, offset, lidx, value, weights, w_pos=None, V_pos=None, pred_init=None):
        offset, lidx = _arr(offset, np.uint64), _arr(lidx, np.uint32)
        value, weights = _arr(value, np.float32), _arr(weights, np.float32)
        w_pos, V_pos = _arr(w_pos, np.int32), _arr(V_pos, np.int32)
        nrows = len(offset) - 1
        pred = np.zeros(nrows, np.float32) if pred_init is None else _arr(pred_init, np.float32).copy()
        npos = 0 if w_pos is None else len(w_pos)
        self._ck(self.L.dfb_predict(self.h, nrows, _p(offset), _p(lidx), _p(value), _p(weights), len(weights),
                                    _p(w_pos), _p(V_pos), npos, _p(pred)))
        return pred

    def calc_grad(self, offset, lidx, value, label, weights, pred, w_pos=None, V_pos=None, grad_init=None):
        offset, lidx = _arr(offset, np.uint64), _arr(lidx, np.uint32)
        value, weights = _arr(value, np.float32), _arr(weights, np.float32)
        label, pred = _arr(label, np.float32), _arr(pred, np.float32)
        w_pos, V_pos = _arr(w_pos, np.int32), _arr(V_pos, np.int32)
        nrows = len(offset) - 1
        grad = np.zeros(len(weights), np.float32) if grad_init is None else _arr(grad_init, np.float32).copy()
        npos = 0 if w_pos is None else len(w_pos)
        self._ck(self.L.dfb_calc_grad(self.h, nrows, _p(offset), _p(lidx), _p(value), _p(label), _p(weights),
                                      len(weights), _p(w_pos), _p(V_pos), npos, _p(pred), _p(grad)))
        return grad

    def evaluate(self, label, pred):
        label, pred = _arr(label, np.float32), _arr(pred, np.float32)
        out = C.c_float()
        self._ck(self.L.dfb_evaluate(self.h, _p(label), _p(pred), len(pred), C.byref(out)))
        return out.value

    def auc(self, label, pred):
        label, pred = _arr(label, np.float32), _arr(pred, np.float32)
        out = C.c_float()
        self._ck(self.L.dfb_auc(self.h, _p(label), _p(pred), len(pred), C.byref(out)))
        return out.value

    # ---- (B) fused step ----
    def train_step(self, offset, lidx, value, label, keys, cnt=None, is_train=True, want_pred=False):
        offset, lidx = _arr(offset, np.uint64), _arr(lidx, np.uint32)
        value, label = _arr(value, np.float32), _arr(label, np.float32)
        keys, cnt = _arr(keys, np.uint64), _arr(cnt, np.float32)
        nrows = len(offset) - 1
        pr = Progress()
        pred = np.zeros(max(nrows, 1), np.float32) if want_pred else None
        self._ck(self.L.dfb_train_step(self.h, nrows, _p(offset), _p(lidx), _p(value), _p(label), _p(keys),
                                       len(keys), _p(cnt), int(is_train), C.byref(pr), _p(pred)))
        return (pr, pred[:nrows]) if want_pred else pr

    # ---- raw ids: GPU localizer + fused step ----
    def localize(self, offset, index, max_index=0xFFFFFFFFFFFFFFFF, want_cnt=True):
        offset, index = _arr(offset, np.uint64), _arr(index, np.uint64)
        nrows = len(offset) - 1
        nnz = int(offset[-1]) if nrows > 0 else 0
        lidx = np.zeros(max(nnz, 1), np.uint32)
        keys = np.zeros(max(nnz, 1), np.uint64)
        cnt = np.zeros(max(nnz, 1), np.float32) if want_cnt else None
        n = C.c_size_t()
        self._ck(self.L.dfb_localize(self.h, nrows, _p(offset), _p(index), max_index, _p(lidx), _p(keys), _p(cnt),
                                     C.byref(n)))
        return lidx[:nnz], keys[:n.value].copy(), (cnt[:n.value].copy() if want_cnt else None)

    def train_step_raw(self, offset, ids, value, label, push_cnt=False, is_train=True, want_pred=False):
        offset, ids = _arr(offset, np.uint64), _arr(ids, np.uint64)
        value, label = _arr(value, np.float32), _arr(label, np.float32)
        nrows = len(offset) - 1
        pr = Progress()
        pred = np.zeros(max(nrows, 1), np.float32) if want_pred else None
        self._ck(self.L.dfb_train_step_raw(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label), int(push_cnt),
                                           int(is_train), C.byref(pr), _p(pred)))
        return (pr, pred[:nrows]) if want_pred else pr

    def train_step_raw_async(self, nrows, offset, ids, value, label, push_cnt=False, is_train=True):
        self._ck(self.L.dfb_train_step_raw_async(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label),
                                                 int(push_cnt), int(is_train)))

    def prefetch_raw(self, nrows, offset, ids, value, label):
        self._ck(self.L.dfb_prefetch_raw(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label)))

    def train_step_raw_dev(self, nrows, nnz, d_offset, d_ids, d_value, d_label, push_cnt=False, is_train=True):
        self._ck(self.L.dfb_train_step_raw_dev(self.h, nrows, nnz, _p(d_offset), _p(d_ids), _p(d_value), _p(d_label),
                                               int(push_cnt), int(is_train)))

    # ---- raw ids: predict steps (the forward pass of a frozen model; nothing of the model is written) ----
    def predict_raw(self, offset, ids, value=None, label=None):
        """one predict step, waited for: (Progress read as train_step_raw reads it, predictions[nrows])"""
        offset, ids = _arr(offset, np.uint64), _arr(ids, np.uint64)
        value, label = _arr(value, np.float32), _arr(label, np.float32)
        nrows = len(offset) - 1
        pred = np.zeros(max(nrows, 1), np.float32)
        self.predict_raw_async(nrows, offset, ids, value, label, pred)
        return self.read_progress(), pred[:nrows]

    def predict_raw_async(self, nrows, offset, ids, value, label, pred_out):
        """raw pointers / arrays, no conversion: pred_out (pinned for an asynchronous copy) is written when the step is
        collected (wait_step / read_progress / sync)"""
        self._ck(self.L.dfb_predict_raw_async(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label), _p(pred_out)))

    def predict_raw_dev(self, nrows, nnz, d_offset, d_ids, d_value, d_label, d_pred_out=None):
        self._ck(self.L.dfb_predict_raw_dev(self.h, nrows, nnz, _p(d_offset), _p(d_ids), _p(d_value), _p(d_label),
                                            _p(d_pred_out)))

    def train_step_async(self, nrows, offset, lidx, value, label, keys, nkeys, cnt=None, is_train=True):
        """raw pointers / arrays, no conversion: for pinned-memory pipelines"""
        self._ck(self.L.dfb_train_step_async(self.h, nrows, _p(offset), _p(lidx), _p(value), _p(label),
                                             _p(keys), nkeys, _p(cnt), int(is_train)))

    def train_step_dev(self, nrows, nnz, d_offset, d_lidx, d_value, d_label, d_keys, nkeys, d_cnt=None,
                       is_train=True):
        self._ck(self.L.dfb_train_step_dev(self.h, nrows, nnz, _p(d_offset), _p(d_lidx), _p(d_value),
                                           _p(d_label), _p(d_keys), nkeys, _p(d_cnt), int(is_train)))

    def sync(self):
        self._ck(self.L.dfb_sync(self.h))

    def wait_step(self):
        pr = Progress()
        self._ck(self.L.dfb_wait_step(self.h, C.byref(pr)))
        return pr

    def profile(self, enable=True):
        self._ck(self.L.dfb_profile(self.h, int(enable)))

    STAGES = ["lookup", "fm", "auc", "csc", "update", "localize", "shard_slice_scatter", "shard_owner_partials",
              "shard_worker_reduce", "shard_owner_updates"]

    def profile_read(self):
        ns = len(self.STAGES)       # DFB_NUM_STAGES
        ms = np.zeros(ns, np.float64)
        cnt = np.zeros(ns, np.uint64)
        self._ck(self.L.dfb_profile_read(self.h, _p(ms), _p(cnt)))
        return {n: dict(ms=float(ms[i]), count=int(cnt[i])) for i, n in enumerate(self.STAGES)}

    def time_mark(self, which):
        self._ck(self.L.dfb_time_mark(self.h, int(which)))

    def time_elapsed_ms(self):
        ms = C.c_float()
        self._ck(self.L.dfb_time_elapsed_ms(self.h, C.byref(ms)))
        return ms.value

    def read_progress(self):
        pr = Progress()
        self._ck(self.L.dfb_read_progress(self.h, C.byref(pr)))
        return pr

    def snapshot(self, save_aux=True):
        n = C.c_size_t()
        self._ck(self.L.dfb_snapshot_size(self.h, int(save_aux), C.byref(n)))
        buf = (C.c_ubyte * max(n.value, 1))()
        self._ck(self.L.dfb_snapshot(self.h, int(save_aux), buf, n.value))
        return C.string_at(buf, n.value)

    def restore(self, blob):
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        aux = C.c_int()
        self._ck(self.L.dfb_restore(self.h, buf, len(blob), C.byref(aux)))
        return bool(aux.value)

    def snapshot_to(self, fileobj, save_aux=True, chunk_bytes=0):
        """stream the snapshot (dfb_snapshot_write) into fileobj.write, at most chunk_bytes per call"""
        failed = []

        def write(_ctx, buf, n):
            try:
                fileobj.write(C.string_at(buf, n))
                return 0
            except Exception as e:     # reported after the C call returns
                failed.append(e)
                return 1
        cb = WRITE_FN(write)
        rc = self.L.dfb_snapshot_write(self.h, int(save_aux), int(chunk_bytes), cb, None)
        if failed:
            raise DfbError(rc, self.L.dfb_last_error(self.h).decode()) from failed[0]
        self._ck(rc)

    def snapshot_begin(self, save_aux=True):
        """freeze the model on the device (dfb_snapshot_begin); the engine may train while the copy is written"""
        f = C.c_void_p()
        self._ck(self.L.dfb_snapshot_begin(self.h, int(save_aux), C.byref(f)))
        self._frozen = [x for x in getattr(self, "_frozen", []) if x.f] + [Frozen(self, f)]
        return self._frozen[-1]

    def id_range(self):
        """the id range learned so far, as a bit count (0: none yet)"""
        b = C.c_int()
        self._ck(self.L.dfb_id_range_get(self.h, C.byref(b)))
        return b.value

    def set_id_range(self, bits):
        self._ck(self.L.dfb_id_range_set(self.h, int(bits)))

    def prune(self, max_count=0.0):
        """drop the entries with w == 0, no V row and fea_cnt <= max_count (dfb_prune), between steps; returns how many
        it dropped"""
        n = C.c_uint64()
        self._ck(self.L.dfb_prune(self.h, float(max_count), C.byref(n)))
        return n.value

    def prune_rare(self, max_count):
        """drop every entry with fea_cnt <= max_count, V rows included, and compact the V-row pool (dfb_prune_rare),
        between steps; returns (entries dropped, V rows freed)"""
        n, v = C.c_uint64(), C.c_uint64()
        self._ck(self.L.dfb_prune_rare(self.h, float(max_count), C.byref(n), C.byref(v)))
        return n.value, v.value

    def restore_from(self, fileobj, part=0, nparts=1, shard=0, nshards=1, chunk_bytes=0):
        """restore (merge) one snapshot stream read from fileobj.read (dfb_restore_read); returns has_aux"""
        failed = []

        def read(_ctx, buf, cap):
            try:
                data = fileobj.read(cap)
                if len(data) > cap:
                    raise ValueError("read returned more than asked for")
                C.memmove(buf, data, len(data))
                return len(data)
            except Exception as e:
                failed.append(e)
                return READ_ERROR
        cb = READ_FN(read)
        aux = C.c_int()
        rc = self.L.dfb_restore_read(self.h, cb, None, part, nparts, shard, nshards, int(chunk_bytes), C.byref(aux))
        if failed:
            raise DfbError(rc, self.L.dfb_last_error(self.h).decode()) from failed[0]
        self._ck(rc)
        return bool(aux.value)

    def read_entries(self, keys):
        keys = _arr(keys, np.uint64)
        n, k = len(keys), self.V_dim
        scal = np.zeros((max(n, 1), 4), np.float32)
        hasv = np.zeros(max(n, 1), np.int32)
        V = np.zeros((max(n, 1), max(k, 1)), np.float32)
        cg = np.zeros((max(n, 1), max(k, 1)), np.float32)
        self._ck(self.L.dfb_read_entries(self.h, _p(keys), n, _p(scal), _p(hasv), _p(V), _p(cg)))
        return scal[:n], hasv[:n], V[:n, :k], cg[:n, :k]

    # ---- sharded building blocks (device pointers / torch tensors) ----
    def dev_feacnt(self, d_keys, n, d_cnt):
        self._ck(self.L.dfb_dev_feacnt(self.h, _p(d_keys), n, _p(d_cnt)))

    def dev_pull_rows(self, d_keys, n, d_w, d_hasv, d_V):
        self._ck(self.L.dfb_dev_pull_rows(self.h, _p(d_keys), n, _p(d_w), _p(d_hasv), _p(d_V)))

    def dev_fm_step(self, nrows, nnz, d_off, d_idx, d_val, d_lab, nkeys, d_w, d_hasv, d_V, is_train, d_gw, d_gV):
        self._ck(self.L.dfb_dev_fm_step(self.h, nrows, nnz, _p(d_off), _p(d_idx), _p(d_val), _p(d_lab), nkeys,
                                        _p(d_w), _p(d_hasv), _p(d_V), int(is_train), _p(d_gw), _p(d_gV)))

    # ---- NVLink peer stores (CUDA IPC) ----
    def peer_alloc(self, nbytes):
        ptr = C.c_void_p()
        handle = (C.c_ubyte * 64)()
        self._ck(self.L.dfb_peer_alloc(self.h, nbytes, C.byref(ptr), handle))
        return ptr.value, bytes(handle)

    def peer_open(self, handle):
        ptr = C.c_void_p()
        buf = (C.c_ubyte * 64).from_buffer_copy(handle)
        self._ck(self.L.dfb_peer_open(self.h, buf, C.byref(ptr)))
        return ptr.value

    def dev_pull_rows_peer(self, d_keys, n, peer_w, peer_hasv, peer_V, d_hasv_local):
        self._ck(self.L.dfb_dev_pull_rows_peer(self.h, _p(d_keys), n, _p(peer_w), _p(peer_hasv), _p(peer_V),
                                               _p(d_hasv_local)))

    def dev_fm_step_peer(self, nrows, nnz, d_off, d_idx, d_val, d_lab, nkeys, d_w, d_hasv, d_V, seg_bounds, peer_gw,
                         peer_gV, first_seg=0):
        nseg = len(peer_gw)
        sb = (C.c_size_t * (nseg + 1))(*[int(x) for x in seg_bounds])
        gw = (C.c_void_p * nseg)(*[int(x) for x in peer_gw])
        gV = (C.c_void_p * nseg)(*[int(x) for x in peer_gV])
        self._ck(self.L.dfb_dev_fm_step_peer(self.h, nrows, nnz, _p(d_off), _p(d_idx), _p(d_val), _p(d_lab), nkeys,
                                             _p(d_w), _p(d_hasv), _p(d_V), nseg, sb, gw, gV, int(first_seg)))

    # ---- the NVLink-sharded store behind the C-ABI (dfb_shard_*) ----
    def shard_init(self, rank, nranks, max_rows, max_nnz, seg_keys=0, seg_nnz=0):
        n = C.c_size_t()
        self._ck(self.L.dfb_shard_init(self.h, rank, nranks, max_rows, max_nnz, seg_keys, seg_nnz, C.byref(n)))
        return n.value

    def shard_export(self):
        """(mailbox device pointer, 64-byte CUDA IPC handle)"""
        ptr = C.c_void_p()
        handle = (C.c_ubyte * 64)()
        self._ck(self.L.dfb_shard_export(self.h, C.byref(ptr), handle))
        return ptr.value, bytes(handle)

    def shard_connect(self, peer_ptrs):
        arr = (C.c_void_p * len(peer_ptrs))(*[C.c_void_p(int(p) if p else 0) for p in peer_ptrs])
        self._ck(self.L.dfb_shard_connect(self.h, arr))

    def shard_step_dev(self, nrows, nnz, d_offset, d_ids, d_value, d_label, push_cnt=False, is_train=True):
        self._ck(self.L.dfb_shard_step_dev(self.h, nrows, nnz, _p(d_offset), _p(d_ids), _p(d_value), _p(d_label),
                                           int(push_cnt), int(is_train)))

    def shard_step_async(self, nrows, offset, ids, value, label, push_cnt=False, is_train=True):
        self._ck(self.L.dfb_shard_step_async(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label),
                                             int(push_cnt), int(is_train)))

    def shard_begin_async(self, nrows, offset, ids, value, label, push_cnt=False, is_train=True):
        self._ck(self.L.dfb_shard_begin_async(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label),
                                              int(push_cnt), int(is_train)))

    def shard_begin_dev(self, nrows, nnz, d_offset, d_ids, d_value, d_label, push_cnt=False, is_train=True):
        self._ck(self.L.dfb_shard_begin_dev(self.h, nrows, nnz, _p(d_offset), _p(d_ids), _p(d_value), _p(d_label),
                                            int(push_cnt), int(is_train)))

    def shard_predict_async(self, nrows, offset, ids, value, label, pred_out):
        self._ck(self.L.dfb_shard_predict_async(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label),
                                                _p(pred_out)))

    def shard_begin_predict_async(self, nrows, offset, ids, value, label, pred_out):
        self._ck(self.L.dfb_shard_begin_predict_async(self.h, nrows, _p(offset), _p(ids), _p(value), _p(label),
                                                      _p(pred_out)))

    def shard_phase(self, phase):
        self._ck(self.L.dfb_shard_phase(self.h, int(phase)))

    def shard_info(self):
        r, n = C.c_int(), C.c_int()
        sk, sn, st = C.c_size_t(), C.c_size_t(), C.c_uint64()
        self._ck(self.L.dfb_shard_info(self.h, C.byref(r), C.byref(n), C.byref(sk), C.byref(sn), C.byref(st)))
        return dict(rank=r.value, nranks=n.value, seg_keys=sk.value, seg_nnz=sn.value, steps=st.value)

    def dev_push_rows(self, d_keys, n, d_gw, d_hasv, d_gV):
        self._ck(self.L.dfb_dev_push_rows(self.h, _p(d_keys), n, _p(d_gw), _p(d_hasv), _p(d_gV)))
