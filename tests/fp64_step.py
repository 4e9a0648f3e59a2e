"""A float64 statement of one SGD step of the reference, with an error bound for every value it predicts, and the harness
that holds an engine's (or the oracle's) step to it.

Semantics (file:line of the reference, as in oracle/fm_oracle.c):
  localize   key = ReverseBytes(id % (2^64 - 1)), unique and ascending                src/data/localizer.cc:22-49
  push_cnt   fea_cnt += count; InitV when w != 0, no V row, fea_cnt > V_threshold        src/sgd/sgd_updater.cc:62-73
  pull       w, and V of the keys that own a row (after the count push)               src/sgd/sgd_updater.cc:32-56
  forward    pred = Xw + .5 sum_f ((XV)_f^2 - (X.X)(V.V)_f), clamped to +-20 unless V_dim = 0   fm_loss.h:67-119
  loss       sum log(1 + exp(-y pred)); p = -y / (1 + exp(y pred))                      loss.h:57-66, fm_loss.h:155-161
  gradients  grad_w = X'p; XXp = (X.X)'p; grad_V = X'diag(p)XV - diag(XXp)V               fm_loss.h:163-199
  update     FTRL on w (l2 term first), then AdaGrad on the V rows pulled               src/sgd/sgd_updater.cc:74-138
  InitV      w left 0, fea_cnt > V_threshold, no row: V_dim rand_r draws, cg = 0, keys ascending (count-push rows
             first)                                                                      src/sgd/sgd_updater.cc:121-147
  penalty    sum l1|w| + .5 l2 w^2 + .5 V_l2 |V|^2 over the pulled weights              src/sgd/sgd_learner.cc:249-273

Everything is computed in float64 (torch, on any device, in row and key chunks of bounded size) from the exact fp32 state
the engine held before the step, so the only differences a correct fp32 step can show are its own roundings.

Error bounds.  u = 2^-24 is the fp32 unit roundoff; 2^-50 is added to it for the float64 statement's own roundings, and
2^-149 (the subnormal spacing) to every rounding for underflow.  gamma(m) = m u / (1 - m u).
  * A sum of m terms in any order (sequential, tree, chunked, atomic) errs by at most gamma(m - 1) sum |t| plus the
    errors of its terms.  This covers every reduction order a kernel may use, including hot keys pre-reduced in chunks.
  * Forward, per row of n nonzeros: |pred - pred64| <= gamma(2n + k + 2) (sum |x w| + .5 (sum_f A_f^2 + Q)) with
    A_f = sum |x V_f| and Q = sum x^2 V_f^2: (XV)_f errs by gamma(n) A_f, its square by gamma(2n + 1) A_f^2, XXVV_f by
    gamma(n + 2) Q_f, their difference by one rounding more, the sum over f by gamma(k - 1), the final add by one.
    The clamp is 1-Lipschitz.  This is order="sorted": the fast forward kernels form XXVV_f per f.
  * order="generic" (k_fm_generic, kernels_fm.cu:457-554: every V_dim > 128, force_generic, the atomic scatter at
    widths other than 8/16/32/64/128, and dfb_predict / dfb_calc_grad) forms the terms differently.  One warp per row,
    lane l holds f = l, l + 32, ... (c = ceil(k / 32) of them):
      - xv_f is a sequential sum over the row's n products a = fl(x V_f) (:498-499): errs by e_f = gamma(n) A_f;
      - s1 = sum_f xv_f^2 is a per-lane fmaf chain over its c values, then a 5-level warp sum (:510-511).  Using xv_f
        for XV_f errs by sum_f e_f (2 |XV_f| + e_f) (first order in e_f: far below gamma(2n + 1) A_f^2 when the x V_f
        cancel), the sum itself by gamma(c + 5) of what it adds;
      - acc2 = Q is a per-lane fmaf chain over all n c of the lane's a^2 (:500), then a 5-level warp sum (:512): a^2
        errs by gamma(2), the chain and the tree by gamma(n c + 5) -- gamma(n c + 7) Q in all.  For n c > 2n + k that
        is more than the sorted statement allows (n = 100 at k = 256; every row at k = 10000);
      - s1 - acc2 and the final add with the linear part (a fmaf chain and a warp sum of n terms: gamma(n) sum |x w|)
        round once each (:513); 0.5 (...) is exact.
    Both forward bounds hold for every order their kernels use; neither is widened to cover the other.
  * |dp/dpred| = s (1 - s), s = sigmoid(pred), is at most 1/4 and falls with |pred|: over pred +- e_pred it is at most
    its value at max(0, |pred| - e_pred).  expf errs by 2 ulp (4u relative), the add and the division by u each:
    e_p = d + gamma(6) (|p| + d) with d = that slope times e_pred.  A row beyond +-20 by more than its bound is clamped
    to exactly +-20 on both sides.  The row loss is 1-Lipschitz in pred; expf, the add and logf (1 ulp) give
    5u + 2u |loss_row| more.  The engine adds row losses in fp32 partials of unknown length: gamma(nrows) of the total.
  * Everything after that -- p XV, the per-key sums, -V XXp, the l2 terms, FTRL and AdaGrad -- is carried as a value
    and an absolute bound through each fp32 operation the update performs (class EV): a product of approximations
    a(1 + .) b(1 + .) errs by |a| e_b + |b| e_a + e_a e_b, a quotient by (e_a + |a / b| e_b) / (|b| - e_b), a square
    root by min(sqrt(e), e / sqrt(a)), and every operation adds u of its magnitude.  The bound of sqrt(sg^2 + g^2) - sg
    is therefore absolute: the difference cancels, and a relative bound of it would be wrong.
  * FTRL's branch: a key whose float64 |z| lies within its bound of l1 is ambiguous -- w may be 0 or the other branch's
    value, and its InitV flag may be either.  They are counted, and the count is capped.
  * The penalty's terms are non-negative and each is evaluated with at most 6 roundings; they are summed in fp32
    partials of at most `pen_partial(n_terms)` terms, then in double.
  * Validation steps: the reference's Pull inserts every key of the batch (model_[key], sgd_updater.cc:32-56), so the
    plugin calls (dfb_pull) do too; the fused entry points insert nothing on a validation step (a missing entry reads
    as w = 0, no V row).  Reference(val_inserts=...) says which of the two a step is held to.

Only tests import this module; it never imports the engine.
"""
import math

import numpy as np
import torch

from oracle.oracle import reverse_bytes_np

F64 = torch.float64
U = 2.0 ** -24 + 2.0 ** -50
ETA = 2.0 ** -149
RAND_A, RAND_C, RAND_MAX = 1103515245, 12345, 2147483647
M32 = np.uint64(0xFFFFFFFF)
# the cap on ambiguous keys, as a fraction of the batch's keys.  The forward bound is a worst case over every summation
# order; at V_dim >= 10 and rows of ~50 nonzeros it leaves up to ~1.5e-3 of the keys of a warm step within their bound of
# l1.  Each of them is still held to one of FTRL's two branches.
AMB_FRAC = 2e-3
# src/sgd/sgd_param.h:94-106
DEFAULTS = dict(l1=1.0, l2=0.0, V_l2=0.01, lr=0.01, lr_beta=1.0, V_lr=0.01, V_lr_beta=1.0, V_init_scale=0.01,
                V_threshold=10, seed=0)
MUTANTS = ("drop_hot_occ", "hot_chunk_dropped", "hot_chunk_twice", "xxp_uses_x", "post_update_V_in_xxp",
           "swap_tile_neighbour", "adagrad_on_new_initv", "no_l2_in_grad_w", "no_clamp")


def gamma(m):
    m = m * U
    return m / (1 - m)


# ---------------------------------------------------------------------------------------------------------------------
# glibc rand_r (stdlib/rand_r.c) restated in numpy, with jump-ahead: row r of the InitV stream starts 3 V_dim r LCG steps
# after the seed (sgd_updater.cc:140-147)
# ---------------------------------------------------------------------------------------------------------------------
def lcg_jump(seed, n):
    """the LCG state n steps after seed (n: int or uint64 array)"""
    n = np.atleast_1d(np.asarray(n, np.uint64)).copy()
    s = np.full(n.shape, seed, np.uint64)
    A, C = np.uint64(RAND_A), np.uint64(RAND_C)
    with np.errstate(over="ignore"):
        while n.any():
            bit = (n & np.uint64(1)).astype(bool)
            s[bit] = (s[bit] * A + C) & M32
            C = (A * C + C) & M32
            A = (A * A) & M32
            n >>= np.uint64(1)
    return s


def _mulmod32(a, s):
    """(a s) mod 2^32 for a < 2^32 and int64 tensors s < 2^32, without overflowing int64"""
    return ((a & 0xFFFF) * s + ((((a >> 16) * s) & 0xFFFF) << 16)) & 0xFFFFFFFF


def initv_rows(seed, start, n, k, scale, device="cpu"):
    """V values of InitV rows start .. start + n - 1 of the stream that begins at seed: float32 [n, k] (on device)"""
    d = torch.device(device)
    todo = (start + torch.arange(n, dtype=torch.int64, device=d)) * (3 * k)
    s = torch.full((n,), int(seed), dtype=torch.int64, device=d)
    A, C = RAND_A, RAND_C
    while bool((todo > 0).any()):
        bit = (todo & 1).bool()
        s = torch.where(bit, (s * A + C) & 0xFFFFFFFF, s)        # A < 2^32: its first power fits; later ones split
        C = (A * C + C) & 0xFFFFFFFF
        A = (A * A) & 0xFFFFFFFF
        todo = todo >> 1
        if A >= 1 << 31:
            break
    while bool((todo > 0).any()):
        bit = (todo & 1).bool()
        s = torch.where(bit, (_mulmod32(torch.full_like(s, A), s) + C) & 0xFFFFFFFF, s)
        C = (A * C + C) & 0xFFFFFFFF
        A = (A * A) & 0xFFFFFFFF
        todo = todo >> 1
    r = torch.empty((n, k), dtype=torch.int64, device=d)
    for f in range(k):
        s = (s * RAND_A + RAND_C) & 0xFFFFFFFF
        x = (s >> 16) % 2048
        s = (s * RAND_A + RAND_C) & 0xFFFFFFFF
        x = (x << 10) ^ ((s >> 16) % 1024)
        s = (s * RAND_A + RAND_C) & 0xFFFFFFFF
        r[:, f] = (x << 10) ^ ((s >> 16) % 1024)
    u = r.to(torch.float32) / np.float32(RAND_MAX)                     # a float division (real_t)
    return ((u.double() - 0.5) * float(np.float32(scale))).float()    # "- 0.5" promotes to double


# ---------------------------------------------------------------------------------------------------------------------
# values with an absolute error bound, through fp32 operations
# ---------------------------------------------------------------------------------------------------------------------
class EV:
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __getitem__(self, i):
        return EV(self.v[i], self.e[i])


def _rnd(v, e):
    """one fp32 rounding of a value known to within e.  Exact inputs (e = 0) whose result float64 holds as an fp32
    value give that value in fp32 too (it is within half a float64 ulp of the exact result, so it is also the nearest
    fp32 value): no error"""
    exact = (e == 0) & (v.float().double() == v)
    return EV(v, torch.where(exact, torch.zeros_like(e), e + U * (v.abs() + e) + ETA))


def ev_add(a, b):
    return _rnd(a.v + b.v, a.e + b.e)


def ev_sub(a, b):
    return _rnd(a.v - b.v, a.e + b.e)


def ev_mul(a, b):
    return _rnd(a.v * b.v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e)


def ev_div(a, b):
    v = a.v / b.v
    den = b.v.abs() - b.e
    e = torch.where(den > 0, (a.e + v.abs() * b.e) / den.clamp_min(1e-300), torch.full_like(v, math.inf))
    return _rnd(v, e)


def ev_sqrt(a):
    v = a.v.clamp_min(0).sqrt()
    e = torch.where(v > 0, torch.minimum(a.e.sqrt(), a.e / v.clamp_min(1e-300)), a.e.sqrt())
    return _rnd(v, e)


def const(x, like):
    return EV(torch.full_like(like, float(np.float32(x))))


def seg_sum(n, idx, t, et, mult=None):
    """sums of terms t (errors et) into n segments: (value, error, |t| sum)"""
    shape = (n,) + tuple(t.shape[1:])
    if mult is not None:
        m = mult.reshape((-1,) + (1,) * (t.dim() - 1))
        t, et = t * m, et * m.abs()
    v = torch.zeros(shape, dtype=F64, device=t.device).index_add_(0, idx, t)
    e = torch.zeros(shape, dtype=F64, device=t.device).index_add_(0, idx, et)
    a = torch.zeros(shape, dtype=F64, device=t.device).index_add_(0, idx, t.abs())
    return v, e, a


def generic_forward_bound(n, k, Lw, A, XV, S1, Q):
    """the bound of k_fm_generic's prediction (module docstring, order="generic") for rows of n nonzeros (float64
    tensor [B]), before the clamp: Lw = sum |x w|, A[B, k] = sum |x V_f|, XV[B, k], S1 = sum_f XV_f^2, Q"""
    c = -(-k // 32)
    e_f = gamma(n)[:, None] * A
    e_sq = (e_f * (2 * XV.abs() + e_f)).sum(1)
    e_s1 = e_sq + gamma(c + 5) * (S1 + e_sq)
    e_Q = gamma(n * c + 7) * Q
    e_d = e_s1 + e_Q + U * ((S1 - Q).abs() + e_s1 + e_Q)
    e_lin = gamma(n) * Lw
    return e_lin + 0.5 * e_d + U * (Lw + 0.5 * (S1 + Q) + e_lin + 0.5 * e_d) + ETA


# ---------------------------------------------------------------------------------------------------------------------
# the reference step
# ---------------------------------------------------------------------------------------------------------------------
def batch_keys(ids):
    """Localizer::Compact: (ascending unique keys, rank of every nonzero, counts)"""
    ids = np.asarray(ids, np.uint64)
    keys, lidx, cnt = np.unique(reverse_bytes_np(np.where(ids == np.uint64(2 ** 64 - 1), np.uint64(0), ids)),
                                return_inverse=True, return_counts=True)
    return keys, lidx.reshape(-1), cnt


class Reference:
    """one SGD step from the pre-step state `pre` = (scal[U, 4] fea_cnt/w/sqrt_g/z, hasv[U] (-1 absent, 0, 1),
    V[U, k], cg[U, k]) of the batch's keys (batch_keys order), and the rng state `seed` before the step.

    mode: "train", "val" (forward, loss, penalty; the batch's absent keys inserted when val_inserts) or "predict"
    (forward only).  mutant: one of MUTANTS, a deliberately wrong variant used to show the comparison's sharpness.
    hot_chunk: the chunk length of the hot-key mutants.  order: "sorted" or "generic", the forward kernel's summation
    order (module docstring).  val_inserts: True for the reference and the plugin calls, False for the fused steps.

    streams: the InitV streams of a step whose keys are owned by S stores by key range (the sharded store): (bounds,
    seeds), bounds[S + 1] cutting the batch's sorted keys into the owners' segments and seeds[S] each owner's rng state
    before the step.  Each owner draws its own stream -- its count-push rows first, then its update's, each in
    ascending key order over its own keys.  `seed` is then unused; None is one stream from `seed` over every key."""

    def __init__(self, batch, hp, pre, seed, push_cnt=False, mode="train", device="cpu", mutant=None, hot_chunk=256,
                 budget=1 << 23, order="sorted", val_inserts=True, streams=None):
        assert mutant is None or mutant in MUTANTS, mutant
        assert order in ("sorted", "generic"), order
        self.order, self.val_inserts = order, bool(val_inserts)
        hp = dict(DEFAULTS, **hp)
        self.hp = {k: (float(np.float32(v)) if isinstance(v, float) else v) for k, v in hp.items()}
        self.k = k = int(hp["V_dim"])
        self.mode, self.push, self.mutant, self.hot_chunk = mode, bool(push_cnt) and mode == "train", mutant, hot_chunk
        self.dev = torch.device(device)
        self.budget = budget
        off, lab, ids, val = batch
        self.off = np.asarray(off, np.int64)
        self.B = len(self.off) - 1
        self.keys, lidx, cnt = batch_keys(ids)
        self.U = Uk = len(self.keys)
        self.cnt = cnt
        if streams is None:
            self.streams = [(0, Uk, int(seed))]
        else:
            bounds, seeds = streams
            assert len(bounds) == len(seeds) + 1 and bounds[0] == 0 and bounds[-1] == Uk, (bounds, Uk)
            self.streams = [(int(a), int(b), int(s)) for a, b, s in zip(bounds[:-1], bounds[1:], seeds)]
        self.seed0 = self.streams[0][2]
        scal, hasv, V, cg = pre
        assert len(hasv) == Uk
        self.absent = hasv < 0
        hv = hasv == 1
        fea = scal[:, 0].astype(np.float32)
        if self.push:
            fea = (fea + cnt.astype(np.float32)).astype(np.float32)
        self.fea1 = fea
        # the count push's InitV (sgd_updater.cc:62-73): ascending keys, at the head of this step's stream
        self.push_initv = np.zeros(Uk, bool)
        if self.push and k > 0:
            self.push_initv = ~hv & (scal[:, 1] != 0) & (fea > np.float32(hp["V_threshold"]))
        self.n_push = int(self.push_initv.sum())
        self.n_push_seg = [int(self.push_initv[a:b].sum()) for a, b, _ in self.streams]
        self.hv_pull = hv | self.push_initv
        Vp = np.where(hv[:, None], V, np.float32(0)).astype(np.float32) if k else np.zeros((Uk, 0), np.float32)
        for a, b, sd in self.streams:
            at, step = a + np.nonzero(self.push_initv[a:b])[0], max(1, budget // max(k, 1))
            for r0 in range(0, len(at), step):
                Vp[at[r0:r0 + step]] = initv_rows(sd, r0, len(at[r0:r0 + step]), k, hp["V_init_scale"],
                                                  device).cpu().numpy()
        cgp = np.where(hv[:, None], cg, np.float32(0)).astype(np.float32) if k else Vp
        if mutant == "swap_tile_neighbour":        # a key's V row swapped with its successor's, mid-tile
            j = self._swap_index()
            Vp[[j, j + 1]] = Vp[[j + 1, j]]
            cgp[[j, j + 1]] = cgp[[j + 1, j]]
        d = self.dev
        self.w0 = torch.from_numpy(scal[:, 1].astype(np.float64)).to(d)
        self.sg0 = torch.from_numpy(scal[:, 2].astype(np.float64)).to(d)
        self.z0 = torch.from_numpy(scal[:, 3].astype(np.float64)).to(d)
        self.Vp = torch.from_numpy(Vp).to(d)
        self.cgp = torch.from_numpy(cgp).to(d)
        self.hvp = torch.from_numpy(self.hv_pull).to(d)
        self.lidx = torch.from_numpy(lidx.astype(np.int64)).to(d)
        lens = np.diff(self.off)
        self.row_of = torch.repeat_interleave(torch.arange(self.B, device=d), torch.from_numpy(lens).to(d))
        self.x = (torch.from_numpy(np.asarray(val, np.float32)).to(d).double() if val is not None else None)
        self.valued = val is not None
        y = torch.from_numpy(np.where(np.asarray(lab) > 0, 1.0, -1.0)).to(d)
        self._forward(y, torch.from_numpy(lens).to(d).double())
        self._penalty()

    def _swap_index(self):
        """a key in the middle of a 32-key tile that owns a V row, and so does its successor"""
        for j in list(range(15, self.U - 1, 32)) + list(range(self.U - 1)):
            if self.hv_pull[j] and self.hv_pull[j + 1]:
                return j
        raise ValueError("no pair of neighbouring V rows to swap")

    def _chunks(self, cum, n, per_item):
        """chunk boundaries over n items whose cumulative element count is cum (len n + 1)"""
        t = max(1, self.budget // max(per_item, 1))
        b = np.concatenate([np.searchsorted(cum, np.arange(0, cum[-1], t), side="right") - 1, np.arange(0, n, t), [n]])
        b = np.unique(np.clip(b, 0, n))
        return [(int(a), int(c)) for a, c in zip(b[:-1], b[1:]) if c > a]

    # ---- forward (fm_loss.h:67-119), loss (loss.h:57-66), p (fm_loss.h:155-161) ----
    def _forward(self, y, n):
        k, d, B = self.k, self.dev, self.B
        lin, Lw = torch.zeros(B, dtype=F64, device=d), torch.zeros(B, dtype=F64, device=d)
        self.XV = torch.zeros((B, k), dtype=F64, device=d)
        A = torch.zeros((B, k), dtype=F64, device=d)
        Q = torch.zeros(B, dtype=F64, device=d)
        for r0, r1 in self._chunks(self.off, B, k + 1):
            a, b = int(self.off[r0]), int(self.off[r1])
            if b == a:
                continue
            seg = self.row_of[a:b] - r0
            kid = self.lidx[a:b]
            x = self.x[a:b] if self.valued else torch.ones(b - a, dtype=F64, device=d)
            t = x * self.w0[kid]
            lin[r0:r1].index_add_(0, seg, t)
            Lw[r0:r1].index_add_(0, seg, t.abs())
            if k:
                xV = x[:, None] * self.Vp[kid].double()
                self.XV[r0:r1].index_add_(0, seg, xV)
                A[r0:r1].index_add_(0, seg, xV.abs())
                Q[r0:r1].index_add_(0, seg, (xV * xV).sum(1))
        if k:
            S1 = (self.XV * self.XV).sum(1)
            pred = lin + 0.5 * (S1 - Q)
            if self.order == "sorted":
                self.e_pred = gamma(2 * n + k + 2) * (Lw + 0.5 * ((A * A).sum(1) + Q)) + ETA
            else:
                self.e_pred = generic_forward_bound(n, k, Lw, A, self.XV, S1, Q)
            if self.mutant != "no_clamp":     # 20 is an fp32 value: a row beyond it by more than its bound is exact
                self.e_pred = torch.where(pred.abs() - self.e_pred >= 20, torch.zeros_like(pred), self.e_pred)
                pred = pred.clamp(-20.0, 20.0)
            self.e_XV = gamma(n)[:, None] * A + ETA
        else:
            pred = lin
            self.e_pred = gamma(n) * Lw + ETA
        self.pred = pred
        zero = (Lw == 0) & ((A.sum(1) + Q == 0) if k else True)      # every term 0: pred is exactly 0
        self.e_pred = torch.where(zero, torch.zeros_like(self.e_pred), self.e_pred)
        ell = torch.logaddexp(torch.zeros_like(pred), -y * pred)
        e_ell = self.e_pred + 5 * U + 2 * U * (ell + self.e_pred + 5 * U) + ETA
        self.loss = float(ell.sum())
        self.e_loss = float(e_ell.sum() + gamma(B) * (ell + e_ell).sum()) + U * (abs(self.loss) + 1e-30)
        p = -y * torch.sigmoid(-y * pred)
        s_near = torch.sigmoid((pred.abs() - self.e_pred).clamp_min(0))    # p' = s (1 - s) is largest nearest 0
        d_p = s_near * (1 - s_near) * self.e_pred
        e_p = d_p + gamma(6) * (p.abs() + d_p) + ETA
        self.p = EV(p, torch.where(zero, torch.zeros_like(e_p), e_p))         # -y / (1 + expf(0)) = -y / 2 exactly

    # ---- penalty of the pulled weights (sgd_learner.cc:249-273) ----
    def _penalty(self):
        hp = self.hp
        w = self.w0
        t = hp["l1"] * w.abs() + 0.5 * hp["l2"] * w * w
        s, n = float(t.sum()), self.U
        if self.k:
            s += float(0.5 * hp["V_l2"] * (self.Vp.double() ** 2).sum(1)[self.hvp].sum())
            n += int(self.hv_pull.sum()) * self.k
        self.pen, self.pen_terms = s, n

    def penalty_bound(self, pen_partial=None):
        m = self.pen_terms if pen_partial is None else min(self.pen_terms, pen_partial(self.U, self.k))
        s = self.pen * (1 + gamma(6))
        return gamma(6) * self.pen + gamma(m) * s + U * s + ETA * self.pen_terms

    # ---- per-key gradients, FTRL, AdaGrad, InitV flags: in key chunks ----
    def key_chunks(self):
        """yields, per chunk [k0, k1) of the batch's keys, the expected state with its bounds"""
        k, d, hp = self.k, self.dev, self.hp
        cnt = torch.from_numpy(self.cnt.astype(np.int64)).to(d)
        cum = np.concatenate([[0], np.cumsum(self.cnt)])
        order = torch.argsort(self.lidx, stable=True)
        hot = int(np.argmax(self.cnt))
        for k0, k1 in self._chunks(cum, self.U, k + 1):
            a, b = int(cum[k0]), int(cum[k1])
            occ = order[a:b]
            kl = self.lidx[occ] - k0
            rows = self.row_of[occ]
            n = k1 - k0
            m = cnt[k0:k1].double()
            out = dict(k0=k0, k1=k1)
            if self.mode != "train":
                yield out
                continue
            mult = None
            if self.mutant in ("drop_hot_occ", "hot_chunk_dropped", "hot_chunk_twice") and k0 <= hot < k1:
                mult = torch.ones(b - a, dtype=F64, device=d)
                j0 = int(cum[hot]) - a
                mh = int(self.cnt[hot])
                if self.mutant == "drop_hot_occ":
                    mult[j0 + mh // 2] = 0
                else:
                    last = ((mh - 1) // self.hot_chunk) * self.hot_chunk
                    mult[j0 + last:j0 + mh] = 0 if self.mutant == "hot_chunk_dropped" else 2
                m = m.clone()
                m[hot - k0] += mh
            x = EV(self.x[occ]) if self.valued else None
            p = self.p[rows]
            # grad_w = X'p (fm_loss.h:163-169); XXp = (X.X)'p (fm_loss.h:171-178)
            tw = ev_mul(x, p) if self.valued else p
            gw = self._reduce(n, kl, tw, m, mult)
            if not self.valued:
                xxp = gw
            elif self.mutant == "xxp_uses_x":
                xxp = gw
            else:
                xxp = self._reduce(n, kl, ev_mul(_rnd(x.v * x.v, x.e), p), m, mult)
            # FTRL (sgd_updater.cc:104-127)
            w0, sg0, z0 = EV(self.w0[k0:k1]), EV(self.sg0[k0:k1]), EV(self.z0[k0:k1])
            G = gw if self.mutant == "no_l2_in_grad_w" else ev_add(gw, ev_mul(w0, const(hp["l2"], w0.v)))
            sg = ev_sqrt(ev_add(ev_mul(sg0, sg0), ev_mul(G, G)))
            lr = const(hp["lr"], w0.v)
            z = ev_sub(z0, ev_sub(G, ev_mul(ev_div(ev_sub(sg, sg0), lr), w0)))
            l1 = hp["l1"]
            num = ev_sub(z, const(l1, z.v)) if l1 == 0 else EV(torch.where(z.v > 0, z.v - l1, z.v + l1),
                                                              z.e + U * (z.v.abs() + z.e) + ETA)
            wnz = ev_div(num, ev_div(ev_add(const(hp["lr_beta"], sg.v), sg), lr))
            zero = z.v.abs() + z.e <= l1
            nz = z.v.abs() - z.e > l1
            amb = ~zero & ~nz
            out.update(gw=gw, xxp=xxp, sg=sg, z=z, wnz=wnz, w_zero=zero, w_amb=amb)
            base = (self.w0[k0:k1] == 0) & ~self.hvp[k0:k1] & torch.from_numpy(
                self.fea1[k0:k1] > np.float32(hp["V_threshold"])).to(d)
            out["initv"] = base & nz if k else torch.zeros_like(nz)
            out["initv_amb"] = base & amb if k else torch.zeros_like(nz)
            if k:
                # grad_V = X'diag(p)XV - diag(XXp)V (fm_loss.h:181-198), then AdaGrad (sgd_updater.cc:129-138)
                pxv = ev_mul(EV(p.v[:, None], p.e[:, None]), EV(self.XV[rows], self.e_XV[rows]))
                xe = EV(x.v[:, None], x.e[:, None]) if self.valued else None
                t = ev_mul(xe, pxv) if self.valued else pxv
                V0 = EV(self.Vp[k0:k1].double())
                cg0 = EV(self.cgp[k0:k1].double())
                hv = self.hvp[k0:k1]
                Vs, cgs, gs = self._adagrad(n, kl, t, xxp, V0, cg0, m, mult)
                if self.mutant == "post_update_V_in_xxp":
                    Vs, cgs, gs = self._adagrad(n, kl, t, xxp, V0, cg0, m, mult, V_term=EV(Vs.v))
                out.update(V=Vs, cg=cgs, hv_pull=hv)
            yield out

    def _reduce(self, n, kl, t, m, mult, extra=None):
        """per-key sums of the terms t (minus `extra`, one more term).  A sum of exact multiples of 1/2 whose absolute
        values add up to at most 2^22 has every partial sum representable in fp32, in any order: it is exact (the
        gradients of a step whose rows all predict 0 are such sums of +-1/2)"""
        v, e, a = seg_sum(n, kl, t.v, t.e, mult)
        inexact = ((t.e != 0) | (2 * t.v != torch.round(2 * t.v))).double()
        off = torch.zeros_like(v).index_add_(0, kl, inexact)
        mm = m
        if extra is not None:
            v, e, a, mm = v - extra.v, e + extra.e, a + extra.v.abs(), m + 1
            off = off + ((extra.e != 0) | (2 * extra.v != torch.round(2 * extra.v))).double()
        while mm.dim() < v.dim():
            mm = mm[:, None]
        exact = (off == 0) & (a <= 2.0 ** 22)
        return EV(v, torch.where(exact, torch.zeros_like(e), e + gamma((mm - 1).clamp_min(0)) * (a + e) + ETA))

    def _adagrad(self, n, kl, t, xxp, V0, cg0, m, mult, V_term=None):
        hp = self.hp
        vx = ev_mul(V0 if V_term is None else V_term, EV(xxp.v[:, None], xxp.e[:, None]))
        gV = self._reduce(n, kl, t, m, mult, extra=vx)
        g = ev_add(gV, ev_mul(const(hp["V_l2"], V0.v), V0))
        cg = ev_sqrt(ev_add(ev_mul(cg0, cg0), ev_mul(g, g)))
        eta = ev_div(const(hp["V_lr"], cg.v), ev_add(cg, const(hp["V_lr_beta"], cg.v)))
        return ev_sub(V0, ev_mul(eta, g)), cg, g


# ---------------------------------------------------------------------------------------------------------------------
# the comparison
# ---------------------------------------------------------------------------------------------------------------------
class Report:
    def __init__(self, what):
        self.what = what
        self.fail = []
        self.n_fail = 0
        self.max_ratio, self.where = 0.0, ""
        self.n_amb = 0
        self.amb_cap = 0

    def bad(self, msg):
        self.n_fail += 1
        if len(self.fail) < 12:
            self.fail.append(msg)

    def within(self, name, got, exp, keys_or_rows, mask=None):
        """|got - exp.v| <= exp.e elementwise (got: float32 tensor, exp: EV), over mask"""
        err = (got.double() - exp.v).abs()
        ratio = torch.where(exp.e > 0, err / exp.e.clamp_min(1e-300), torch.where(err == 0, 0.0, math.inf))
        if mask is not None:
            m = mask
            while m.dim() < ratio.dim():
                m = m[:, None]
            ratio = torch.where(m, ratio, torch.zeros_like(ratio))
        ratio = torch.nan_to_num(ratio, nan=math.inf)
        r = float(ratio.max()) if ratio.numel() else 0.0
        if r > self.max_ratio:
            self.max_ratio = r
            self.where = name
        bad = ratio > 1
        if bad.any():
            idx = torch.nonzero(bad)
            self.n_fail += int(idx.shape[0]) - 1
            i = tuple(int(v) for v in idx[0])
            self.bad(f"{name}: {int(idx.shape[0])} outside their bound; first at {keys_or_rows(i)}: got "
                     f"{float(got[i]):.9g}, want {float(exp.v[i]):.9g} +- {float(exp.e[i]):.3g}")

    def exact(self, name, ok, detail=""):
        if not ok:
            self.bad(f"{name} {detail}")

    def ok(self):
        return self.n_fail == 0

    def summary(self):
        return (f"{self.what}: max error/bound {self.max_ratio:.3g} ({self.where}), ambiguous keys {self.n_amb} "
                f"(cap {self.amb_cap})")

    def assert_ok(self):
        assert self.ok(), self.summary() + f"; {self.n_fail} failures:\n  " + "\n  ".join(self.fail)


def pen_partial_engine(n_keys, k):
    """the longest fp32 partial of the engine's penalty sums: a lane adds the terms of the keys its warp visits in a
    grid-stride loop, and every such launch has at least min(n / 32, 4096) warps -- so at most max(32, n / 4096) keys,
    and at most V_dim + 1 terms per key, reach one partial before the warp sum (5 levels) and the double atomics"""
    return max(32, -(-n_keys // 4096)) * (k + 1) + 5


def _grid_warps(nwarps_needed, num_sms):
    """the warps of a grid_warps(nwarps_needed, 8, num_sms * 8) launch of 256-thread blocks (kernels_table.cu:1160)"""
    return min(max(1, -(-nwarps_needed // 8)), num_sms * 8) * 8


def pen_partial_warp_per_key(num_sms):
    """k_update_dense_generic (kernels_table.cu:326-369, launched at :1286) and k_penalty (:412-432, launched at
    :1301): grid_warps(n, 8, num_sms * 8), one warp per key in a grid-stride loop.  Lane 0 adds pen_w and each lane
    its ceil(k / 32) terms 0.5 V_l2 v^2 of every key its warp visits into one fp32 partial; then the warp sum (5 levels)
    and a double atomic.  (pen_partial_engine bounds this too whenever num_sms >= 64; this is the launch's own count.)"""
    def m(n_keys, k):
        keys = -(-n_keys // _grid_warps(n_keys, num_sms))
        return keys * (1 + -(-k // 32)) + 5
    return m


def pen_partial_update_fast(num_sms):
    """k_update_fast<K> at the exact widths K = V_dim (kernels_table.cu:273-323, launched at :1281): G = 128 / K keys
    per warp iteration, a group of K / 4 lanes per key; grid_warps(ceil(n / G), 8, num_sms * 8).  The group's first
    lane adds pen_w, every lane adds 0.5 V_l2 (v.x^2 + v.y^2 + v.z^2 + v.w^2) -- four terms summed (3 adds) and scaled
    (1 rounding) before they join the partial: at most 5 terms per key visited, each through at most 4 roundings
    more, then the warp sum (5 levels) and a double atomic"""
    def m(n_keys, k):
        G = 128 // k
        tiles = -(-n_keys // G)
        it = -(-tiles // _grid_warps(tiles, num_sms))
        return it * 5 + 4 + 5
    return m


def pen_partial_bwd_worker(num_sms):
    """k_bwd_update<K, VAL, APPLY = false> (kernels_table.cu:714-1060, launched by launch_bwd_dense at :1469): the
    sharded store's worker emitting gradient rows at the exact widths, grid_warps(ceil(n / 32), 8, num_sms * 8), 32 keys
    per warp iteration.  A lane adds pen_w of its own key (phase A), 0.5 V_l2 (v.x^2 + .. + v.w^2) of the key its group
    holds in each of the K / 4 passes (phase B), and, on the first group, that term of every hot key (more than 64
    occurrences; at most 32): 1 + K / 4 + 32 terms per iteration, four squares summed before they join, then the warp
    sum (5 levels) and a double atomic"""
    def m(n_keys, k):
        tiles = -(-n_keys // 32)
        it = -(-tiles // _grid_warps(tiles, num_sms))
        return it * (1 + k // 4 + 32) + 4 + 5
    return m


def check(ref, pre, post, obs, what="step", pen_partial=None, amb_frac=AMB_FRAC):
    """hold one step's result to the reference.  pre / post: the state of ref's keys before / after (read_entries
    layout); obs: dict with any of loss, penalty, auc, nrows, new_keys, new_vrows, n_keys_delta, n_vrows_delta,
    rng_after, pred (the step's returned predictions), label (for the AUC).  Returns a Report."""
    R = Report(what)
    k, d, U_ = ref.k, ref.dev, ref.U
    keys = ref.keys
    R.amb_cap = max(2, int(math.ceil(amb_frac * U_)))
    scal1, hv1, V1, cg1 = post
    scal0, hv0, V0, cg0 = pre

    def at_key(i):
        return f"key {int(keys[ref_k0 + i[0]]):#018x}" + (f"[{i[1]}]" if len(i) > 1 else "")

    # ---- scalars of Progress ----
    if "nrows" in obs:
        R.exact("nrows", obs["nrows"] == ref.B, f"{obs['nrows']} vs {ref.B}")
    if "loss" in obs:
        e = abs(obs["loss"] - ref.loss)
        R.max_ratio, R.where = max((R.max_ratio, R.where), (e / ref.e_loss, "loss"))
        R.exact("loss", e <= ref.e_loss, f"{obs['loss']!r} vs {ref.loss!r} +- {ref.e_loss:.3g}")
    if "penalty" in obs:
        want = ref.pen if ref.mode != "predict" else 0.0
        eb = ref.penalty_bound(pen_partial) if ref.mode != "predict" else 0.0
        e = abs(obs["penalty"] - want)
        if eb > 0:
            R.max_ratio, R.where = max((R.max_ratio, R.where), (e / eb, "penalty"))
        R.exact("penalty", e <= eb, f"{obs['penalty']!r} vs {want!r} +- {eb:.3g}")
    if obs.get("pred") is not None:
        got = torch.from_numpy(np.asarray(obs["pred"], np.float32)).to(d)
        R.within("pred", got, EV(ref.pred, ref.e_pred), lambda i: f"row {i[0]}")
        if "auc" in obs and "label" in obs:
            R.exact("auc", np.float32(obs["auc"]) == np.float32(auc64(obs["label"], obs["pred"])),
                    f"{obs['auc']} vs float64 AUC of the returned predictions {auc64(obs['label'], obs['pred'])}")
    inserted = ref.mode == "train" or (ref.mode == "val" and ref.val_inserts)
    n_new_keys = int(ref.absent.sum()) if inserted else 0
    if "new_keys" in obs:
        R.exact("new_keys", obs["new_keys"] == n_new_keys, f"{obs['new_keys']} vs {n_new_keys}")
    if "n_keys_delta" in obs:
        R.exact("n_keys", obs["n_keys_delta"] == n_new_keys, f"grew by {obs['n_keys_delta']}, want {n_new_keys}")

    # ---- exact: fea_cnt, presence, V-row pattern ----
    want_fea = ref.fea1 if ref.mode == "train" else scal0[:, 0]
    bad = np.nonzero(scal1[:, 0] != want_fea)[0]
    R.exact("fea_cnt", len(bad) == 0, f"{len(bad)} differ, first key {int(keys[bad[0]]):#018x}: "
            f"{scal1[bad[0], 0]} vs {want_fea[bad[0]]}" if len(bad) else "")
    if ref.mode != "train":
        want_hv = np.where(ref.absent & inserted, 0, hv0)
        same = (hv1 == want_hv) & (scal1 == np.where(ref.absent[:, None] & inserted, 0, scal0)).all(1)
        if k:
            same &= (V1 == V0).all(1) & (cg1 == cg0).all(1)
        bad = np.nonzero(~same)[0]
        R.exact("state", len(bad) == 0, f"{len(bad)} keys changed by a {ref.mode} step, first "
                f"{int(keys[bad[0]]):#018x}" if len(bad) else "")
        if "new_vrows" in obs:
            R.exact("new_vrows", obs["new_vrows"] == 0, f"{obs['new_vrows']}")
        if "rng_after" in obs:
            got = _per_stream(R, ref, obs["rng_after"])
            want = [sd for _, _, sd in ref.streams]
            R.exact("rng", got == want, f"{got} vs {want}")
        return R

    # ---- training: every key against its bounds, in chunks ----
    new_rows = []          # (index, certain) of rows the update's InitV gave
    amb_all = np.zeros(U_, bool)
    for ch in ref.key_chunks():
        ref_k0 = k0 = ch["k0"]
        k1 = ch["k1"]
        s1 = torch.from_numpy(scal1[k0:k1]).to(d)
        R.within("sqrt_g", s1[:, 2], ch["sg"], at_key)
        R.within("z", s1[:, 3], ch["z"], at_key)
        amb, zero = ch["w_amb"], ch["w_zero"]
        w1 = s1[:, 1]
        R.within("w", w1, ch["wnz"], at_key, mask=~zero & ~amb)
        nz = zero & (w1 != 0)
        R.exact("w", not bool(nz.any()), f"{int(nz.sum())} keys with |z| below l1 by more than its bound have w != 0")
        amb_ok = (w1 == 0) | ((w1.double() - ch["wnz"].v).abs() <= ch["wnz"].e)
        R.exact("w (ambiguous key)", bool((amb_ok | ~amb).all()), "")
        R.n_amb += int(amb.sum())
        amb_all[k0:k1] = ch["initv_amb"].cpu().numpy()
        if k:
            hvp = ch["hv_pull"]
            V1c, cg1c = torch.from_numpy(V1[k0:k1]).to(d), torch.from_numpy(cg1[k0:k1]).to(d)
            R.within("V", V1c, ch["V"], at_key, mask=hvp)
            R.within("cg", cg1c, ch["cg"], at_key, mask=hvp)
            hv_after = torch.from_numpy(hv1[k0:k1] == 1).to(d)
            got_new = hv_after & ~hvp
            flag, flag_amb = ch["initv"], ch["initv_amb"]
            wrong = (got_new != flag) & ~flag_amb
            if bool(wrong.any()):
                i = int(torch.nonzero(wrong)[0])
                R.bad(f"V-row pattern: {int(wrong.sum())} keys differ, first key {int(keys[k0 + i]):#018x}: has a row "
                      f"{bool(got_new[i])}, InitV due {bool(flag[i])}")
            lost = hvp & ~hv_after
            R.exact("V rows lost", not bool(lost.any()), f"{int(lost.sum())}")
            new_rows.append(torch.nonzero(got_new).flatten().cpu().numpy() + k0)
    R.exact("ambiguous keys", R.n_amb <= R.amb_cap, f"{R.n_amb} > cap {R.amb_cap}")
    ref_k0 = 0

    # ---- the InitV streams (one per owner): count-push rows first, then the update's, each in ascending key order ----
    if k:
        upd = np.concatenate(new_rows) if new_rows else np.zeros(0, np.int64)
        n_new = ref.n_push + len(upd)
        if "new_vrows" in obs:
            R.exact("new_vrows", obs["new_vrows"] == n_new, f"{obs['new_vrows']} vs {n_new} new rows in the table")
        if "n_vrows_delta" in obs:
            R.exact("n_vrows", obs["n_vrows_delta"] == n_new, f"grew by {obs['n_vrows_delta']}, want {n_new}")
        got_rng = _per_stream(R, ref, obs["rng_after"]) if "rng_after" in obs else None
        badv, first = 0, ""
        step = max(1, ref.budget // max(k, 1))          # the stream's rows in chunks of bounded size
        for j, ((a, b, sd), n_push) in enumerate(zip(ref.streams, ref.n_push_seg)):
            mine = upd[(upd >= a) & (upd < b)]
            if got_rng is not None:
                n_s = n_push + len(mine)
                want = int(lcg_jump(sd, 3 * k * n_s)[0])
                R.exact("rng", got_rng[j] == want, f"stream {j}: {got_rng[j]} vs seed jumped by 3 V_dim {n_s} = {want}")
            for r0 in range(0, len(mine), step):
                rows = mine[r0:r0 + step]
                Vw = initv_rows(sd, n_push + r0, len(rows), k, ref.hp["V_init_scale"], d).cpu().numpy()
                if ref.mutant == "adagrad_on_new_initv":
                    Vw = _adagrad_fresh(ref.hp, Vw)
                bad = np.nonzero(~((V1[rows] == Vw).all(1) & (cg1[rows] == 0).all(1)))[0]
                if len(bad) and not badv:
                    first = f"key {int(keys[rows[bad[0]]]):#018x}: {V1[rows[bad[0]]][:4]} vs {Vw[bad[0]][:4]}"
                badv += len(bad)
        R.exact("InitV values", badv == 0, f"{badv} of {len(upd)} new rows differ from the stream, first {first}")
    elif "rng_after" in obs:
        got = _per_stream(R, ref, obs["rng_after"])
        R.exact("rng", got == [sd for _, _, sd in ref.streams], "")
    return R


def _per_stream(R, ref, rng_after):
    """the observed rng state of every InitV stream: one value, or one per owner when the step has several streams"""
    got = [int(x) for x in np.atleast_1d(np.asarray(rng_after, np.int64))]
    R.exact("rng streams", len(got) == len(ref.streams), f"{len(got)} rng states for {len(ref.streams)} streams")
    return (got + [None] * len(ref.streams))[:len(ref.streams)]


def _adagrad_fresh(hp, V):
    """AdaGrad with a zero loss gradient on a fresh row (the adagrad_on_new_initv mutant), in float32 as the update"""
    V = V.astype(np.float32)
    g = (np.float32(hp["V_l2"]) * V).astype(np.float32)
    cg = np.sqrt(g * g).astype(np.float32)
    eta = (np.float32(hp["V_lr"]) / (cg + np.float32(hp["V_lr_beta"]))).astype(np.float32)
    return (V - eta * g).astype(np.float32)


def assert_unchanged(before, after, keys, what):
    """keys outside a step's batch: bit for bit what they were"""
    for name, a, b in zip(("scalars", "hasv", "V", "cg"), before, after):
        bad = np.nonzero(~(np.asarray(a) == np.asarray(b)).reshape(len(keys), -1).all(1))[0]
        assert len(bad) == 0, f"{what}: {name} of {len(bad)} keys outside the batch changed, first {int(keys[bad[0]]):#018x}"


def auc64(label, pred):
    """BinClassMetric::AUC (src/loss/bin_class_metric.h:35-56) in float64: a stable sort by prediction"""
    label, pred = np.asarray(label), np.asarray(pred)
    pos = label[np.argsort(pred, kind="stable")] > 0
    n, tp = len(pred), int(pos.sum())
    if tp == 0 or tp == n:
        return 1.0
    area = float(np.cumsum(pos)[~pos].sum()) / (float(tp) * float(n - tp))
    return (1.0 - area if area < 0.5 else area) * n
