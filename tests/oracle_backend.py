"""CPU backend for difacto_b200.sharded.ShardedStore built on the oracle -- TEST INFRASTRUCTURE.

It lets the world_size-2 gloo tests exercise the sharding protocol (key-range partition, count
exchange, all_to_all_v splits, per-source application order) without a GPU.  The product only
ever constructs CudaBackend."""
import numpy as np
import torch

from oracle import oracle as O


def _keys_np(t):
    return t.numpy().view(np.uint64) if len(t) else np.zeros(0, np.uint64)


class OracleBackend:
    def __init__(self, **kw):
        self.M = O.Oracle(**kw)
        self.V_dim = self.M.V_dim
        self.ks = (self.V_dim + 3) // 4 * 4
        self.progress = np.zeros(5, np.float64)   # loss, penalty, auc, nnz_w, nrows

    def empty(self, shape, dtype):
        return torch.zeros(shape, dtype=dtype)

    def feacnt(self, keys, cnt):
        if len(keys):
            self.M.update_feacnt(_keys_np(keys), cnt.numpy())

    def pull_rows(self, keys, w, hasv, V):
        k = self.V_dim
        if not len(keys):
            return
        n = len(keys)
        vals, lens = self.M.get(_keys_np(keys))
        if not k:                                   # V_dim 0: one value per key, no lens
            lens = np.ones(n, np.int32)
        start = np.cumsum(lens) - lens
        w[:n] = torch.from_numpy(vals[start])
        has = lens > 1
        hasv[:n] = torch.from_numpy(np.where(has, 1, -1).astype(np.int32))
        if has.any():
            V[torch.from_numpy(np.nonzero(has)[0]), :k] = torch.from_numpy(vals[start[has, None] + 1 + np.arange(k)])

    def _ragged(self, w, hasv, V):
        k = self.V_dim
        U = len(w)
        if k == 0:
            return w.numpy().copy(), None, None, np.zeros(0, np.int32)
        lens = np.where(hasv.numpy() > 0, k + 1, 1).astype(np.int32)
        w_pos, V_pos = O.get_pos(lens)
        vals = np.zeros(int(lens.sum()), np.float32)
        vals[w_pos] = w.numpy()
        m = V_pos >= 0
        vals[V_pos[m, None] + np.arange(k)] = V[:U, :k].numpy()[m]
        return vals, w_pos, V_pos, lens

    def fm_step(self, batch, w, hasv, V, is_train, gw, gV):
        k = self.V_dim
        off = batch["off"].numpy().view(np.uint64)
        lidx = batch["lidx"].numpy().view(np.uint32)
        val = batch["val"].numpy() if batch.get("val") is not None else None
        lab = batch["lab"].numpy()
        vals, w_pos, V_pos, lens = self._ragged(w[:batch["U"]], hasv[:batch["U"]], V[:batch["U"]])
        pred = O.fm_predict(k, off, lidx, val, vals, w_pos, V_pos)
        self.progress[0] += O.evaluate(lab, pred)
        self.progress[1] += O.penalty(self.M.param, vals, w_pos, V_pos)
        self.progress[2] += O.auc(lab, pred)
        self.progress[4] += len(lab)
        if not is_train:
            return
        g = O.fm_calc_grad(k, off, lidx, val, lab, vals, pred, w_pos, V_pos)
        if k == 0:
            gw[:] = torch.from_numpy(g)
            return
        gw[:] = torch.from_numpy(g[w_pos])
        m = np.nonzero(V_pos >= 0)[0]
        gV[torch.from_numpy(m), :k] = torch.from_numpy(g[V_pos[m, None] + np.arange(k)])

    def push_rows(self, keys, gw, hasv, gV):
        if not len(keys):
            return
        k = self.V_dim
        if k == 0:
            self.M.update_grad(_keys_np(keys), gw.numpy(), np.zeros(0, np.int32))
            return
        lens = np.where(hasv.numpy() > 0, k + 1, 1).astype(np.int32)
        w_pos, V_pos = O.get_pos(lens)
        g = np.zeros(int(lens.sum()), np.float32)
        g[w_pos] = gw.numpy()
        m = V_pos >= 0
        g[V_pos[m, None] + np.arange(k)] = gV[:, :k].numpy()[m]
        self.M.update_grad(_keys_np(keys), g, lens)
