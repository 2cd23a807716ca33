"""Float64 reference of the MLP layers and of one train step's gradients, recomputed from the values the GPU itself used.

Every stage starts from the inputs its kernel actually read (``deep_input()``, ``hidden_output()`` of the source layers, the fp32
parameters), so each kernel is judged on its own error and not on drift from the layers before it, and no relu gate can flip
between the two sides.  Gradients are read through the public API: with SGD at a learning rate of 2^24, one step moves every
parameter by exactly 2^24 * g up to one fp32 rounding of the result, so g = (w_before - w_after) / 2^24 (``probe_step``).

Each compared tensor is held to two criteria:

1. elementwise, uncalibrated: ``|gpu - ref| <= C * M + 4 ulp(ref) + slack``.  M is the same computation run on absolute values
   (|W|, |inp|, |act'|, |gamma * inv|, |dlogit|), C a worst-case bound of the engine's product and fp32 summation error
   (``c_gemm``) times the number of GEMMs on the path.  Catches gross faults: a missing k-block, a stale row, a wrong tile, NaN.
2. statistical, per 128 x 128 output tile: ``RMS(|gpu - ref| / R) <= tau``, R = sqrt(sum_k (a_ik b_kj)^2) of the reduction.  For
   gradients, R also carries the R of the operands that earlier GEMMs of the backward produced (R^2 of a * b adds a^2 R_b^2),
   so cancellation in a data gradient does not count against the GEMM that reads it.  Checking each tile separately keeps a
   fault confined to the ragged last tile from being diluted by the healthy ones.

The numpy emulation of the engines (``emulated_gemm``: bf16 / tf32 rounding, the three-pass hi / lo products with fp32
accumulation) lets the CPU suite pin the checker down before any GPU runs: the healthy engines pass, planted defects fail.
"""
import numpy as np

from oracle.model import act_fwd as _oracle_act_fwd, drop_keep, layer_sources

U = 2.0 ** -24
GAMMA_SCALE = float(np.float32(0.99950037468777))        # 1 / sqrt(1 + 1e-3), the fp32 constant of the kernels
SELU_A, SELU_S = 1.6732632423543772, 1.0507009873554805
RELU_FAMILY = ("relu", "relu6", "leaky_relu", "crelu")
LIP = dict(sigmoid=0.25, selu=SELU_A * SELU_S)           # Lipschitz constant of the activation (1 for the others)
DLIP = dict(sigmoid=1.0, tanh=2.0, elu=1.0, selu=1.0, softplus=1.0, softsign=2.0)   # max |d act'(a) / da| of act_bwd_from_a
TILE = 128


# ------------------------------------------------------------------------------------------------ engine emulation
def bf16_round(x):
    """Round to the nearest bf16 (ties to even) on the fp32 bit pattern; returned as float32."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def tf32_round(x):
    """Round to the nearest tf32 (10 explicit mantissa bits, ties away from zero, as cvt.rna.tf32.f32); returned as float32."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x1000) & 0xFFFFE000
    return b.astype(np.uint32).view(np.float32)


def split_hi_lo(x, rnd):
    x = np.asarray(x, dtype=np.float32)
    hi = rnd(x)
    return hi, rnd(x - hi)


def emulated_gemm(a, b, engine, single_pass=False, drop_lohi_kblock=None, kblock=32):
    """a @ b as the engine computes it: ffma = fp32 products and sums; tc3x / bf16x3 = lo*hi + hi*lo + hi*hi of the tf32 / bf16
    hi / lo copies (every product exact in fp32) with fp32 accumulation.  single_pass: hi*hi only (tc1x and a bf16 single pass);
    drop_lohi_kblock: leave out the lo*hi term of that k-block (a planted defect)."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    if engine == "ffma":
        return (a @ b).astype(np.float64)
    ah, al = split_hi_lo(a, bf16_round if engine == "bf16x3" else tf32_round)
    bh, bl = split_hi_lo(b, bf16_round if engine == "bf16x3" else tf32_round)
    out = ah @ bh
    if not single_pass:
        if drop_lohi_kblock is not None:
            al = al.copy()
            al[:, drop_lohi_kblock * kblock:(drop_lohi_kblock + 1) * kblock] = 0
        out = al @ bh + ah @ bl + out
    return out.astype(np.float64)


def c_gemm(engine, K):
    """Worst-case relative error (against the sum of |products|) of one K-long dot product of the engine, fp32 sums included."""
    if engine == "ffma":
        return (K + 2) * U
    if engine == "tc3x":
        return 2.0 ** -19 + K * 2.0 ** -23
    if engine == "bf16x3":
        return 2.0 ** -15 + K * 2.0 ** -23
    raise ValueError(engine)


# ------------------------------------------------------------------------------------------------ activations
def act_fwd(name, z):
    return np.maximum(z, 0) if name == "crelu" else _oracle_act_fwd(name, z)      # (crelu layers run as relu of twice the width)


def act_bwd_from_a(name, a):
    """d act / d z from the post-activation value a, the formulas of csrc/gemm.cuh act_bwd, in float64."""
    if name in ("relu", "crelu"):
        return (a > 0).astype(np.float64)
    if name == "relu6":
        return ((a > 0) & (a < 6)).astype(np.float64)
    if name == "sigmoid":
        return a * (1 - a)
    if name == "tanh":
        return 1 - a * a
    if name == "leaky_relu":
        return np.where(a > 0, 1.0, 0.2)
    if name == "elu":
        return np.where(a > 0, 1.0, a + 1.0)
    if name == "selu":
        return np.where(a > 0, SELU_S, a + SELU_S * SELU_A)
    if name == "softplus":
        return 1 - np.exp(-a)
    if name == "softsign":
        return (1 - np.abs(a)) ** 2
    raise ValueError(name)


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


# ------------------------------------------------------------------------------------------------ the two criteria
class Check(object):
    """Result of comparing one tensor: worst1 = max |gpu - ref| / bound (criterion 1 passes at <= 1), worst2 = worst tile RMS of
    |gpu - ref| / R (criterion 2 passes at <= tau)."""

    def __init__(self, name, worst1, where1, worst2, tile2):
        self.name, self.worst1, self.where1, self.worst2, self.tile2 = name, worst1, where1, worst2, tile2

    def __repr__(self):
        return "%s: criterion 1 %.3g at %s, criterion 2 %.3g in tile %s" % (self.name, self.worst1, self.where1, self.worst2, self.tile2)


def compare(name, gpu, ref, M, R, C, slack=0.0):
    gpu, ref = np.asarray(gpu, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert gpu.shape == ref.shape, (name, gpu.shape, ref.shape)
    if gpu.ndim == 1:
        gpu, ref, M = gpu[None], ref[None], np.asarray(M, dtype=np.float64)[None]
        R = None if R is None else np.asarray(R, dtype=np.float64)[None]
    if gpu.size == 0:
        return Check(name, 0.0, None, 0.0, None)
    err = np.abs(gpu - ref)
    bound = C * np.broadcast_to(M, err.shape) + 4 * ulp32(ref) + slack
    with np.errstate(divide="ignore", invalid="ignore"):
        r1 = np.where(err == 0, 0.0, err / bound)
    r1[~np.isfinite(gpu)] = np.inf
    i1 = np.unravel_index(int(np.argmax(r1)), r1.shape)
    worst2, tile2 = 0.0, None
    if R is None:                                       # (criterion 1 only)
        return Check(name, float(r1[i1]), tuple(int(i) for i in i1), worst2, tile2)
    R = np.broadcast_to(R, err.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(R > 0, err / R, 0.0)
    ratio[~np.isfinite(gpu)] = np.inf
    for r0 in range(0, err.shape[0], TILE):
        for c0 in range(0, err.shape[1], TILE):
            cnt = int((R[r0:r0 + TILE, c0:c0 + TILE] > 0).sum())
            if cnt:
                rms = float(np.sqrt((ratio[r0:r0 + TILE, c0:c0 + TILE] ** 2).sum() / cnt))
                if not rms <= worst2:
                    worst2, tile2 = rms, (r0 // TILE, c0 // TILE)
    return Check(name, float(r1[i1]), tuple(int(i) for i in i1), worst2, tile2)


# ------------------------------------------------------------------------------------------------ reading the GPU
LR_PROBE = 2.0 ** 24


def probe_step(pm, batch, params, split=False):
    """Upload `params`, run one SGD step (learning rate 2^24) and return (gradients, parameters after) in float64.  split: the
    unfused wd_step_backward + wd_step_apply instead of wd_train_step."""
    for name, v in params.items():
        pm.set_tensor(name, v)
    if split:
        pm.step_backward(batch)
        pm.step_apply()
    else:
        pm.train_step(batch)
    after = {n: pm.get_tensor(n) for n in params}
    return {n: (params[n].astype(np.float64) - after[n]) / LR_PROBE for n in params}, after


def gpu_forward_values(pm, B):
    """The step's forward values as the GPU holds them: deep input [B, d0_phys] and, per tower, every hidden output [B, N_phys]."""
    X0 = pm.deep_input(B).astype(np.float64)
    H = [[pm.hidden_output(t, l, B).astype(np.float64) for l in range(len(tw["hidden"]))] for t, tw in enumerate(pm.plan.towers)]
    return X0, H


def x0_logical(plan, X0p):
    return np.concatenate([X0p[:, po:po + w] for _, (lo, po, w) in plan.deep_layout.items()], axis=1)


def x0_padding_mask(plan):
    keep = np.zeros(plan.d0_phys, dtype=bool)
    for _, (lo, po, w) in plan.deep_layout.items():
        keep[po:po + w] = True
    return ~keep


def scope(t, l, L):
    return "dnn/dnn_%d/" % (t + 1) + ("hiddenlayer_%d" % l if l < L else "logits")


# ------------------------------------------------------------------------------------------------ the reference step
class StepRef(object):
    """Reference of one step on the GPU's own forward values.

    pm: the WideDeepModel after the step; batch: the Batch it ran; params: fp32 parameters it started from; step: the dropout counter
    of the step (train steps before it; None for a forward without dropout); engine: the GEMM engine the C bounds are for.
    """

    def __init__(self, pm, batch, params, engine, step=None):
        self.plan, self.engine, self.params = pm.plan, engine, {k: np.asarray(v, dtype=np.float64) for k, v in params.items()}
        plan = self.plan
        self.B = B = batch.batch_size
        self.X0p, self.H = gpu_forward_values(pm, B) if plan.use_deep else (None, [])
        self.X0 = x0_logical(plan, self.X0p) if plan.use_deep else None
        self.offs, self.ids = pm.column_ids()
        self.label = batch.label.astype(np.float64)
        self.weight = np.ones(B) if batch.weight is None else batch.weight.astype(np.float64)
        self.act, self.bn = plan.activation, plan.batch_norm
        self.rate = plan.dropout if step is not None else 0.0
        self.step = step

    # ---- helpers
    def _col_ids(self, col):
        """(row index per id, id) of one categorical column of the batch."""
        C = len(self.plan.columns)
        ci = self.plan._col_index[id(col)]
        s, e = self.offs[ci:self.B * C:C], self.offs[ci + 1:self.B * C + 1:C]
        cnt = e - s
        rows = np.repeat(np.arange(self.B), cnt)
        pos = np.concatenate([np.arange(a, b) for a, b in zip(s, e)]) if len(s) else np.zeros(0, dtype=np.int64)
        return rows, self.ids[pos.astype(np.int64)], cnt

    def _bag_scale(self, cnt):
        """The mean combiner's factor of each bag, from its id count."""
        return 1.0 / np.maximum(cnt, 1)

    def _keep(self, t, l, width):
        if self.rate <= 0:
            return None
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(self.rate)))
        return drop_keep(self.plan.dropout_seed, self.step, t * 64 + l, self.B, width, self.rate).astype(np.float64) * scale

    def _layer_params(self, t, l, L):
        p = self.params
        sc = scope(t, l, L)
        W, b = p[sc + "/kernel"], p[sc + "/bias"]
        if l < L and self.act == "crelu":
            W, b = np.concatenate([W, -W], axis=1), np.concatenate([b, -b])
        gp = be = None
        if l < L and self.bn:
            gp = (p[sc + "/batch_normalization/gamma"].astype(np.float32) * np.float32(GAMMA_SCALE)).astype(np.float64)
            be = p[sc + "/batch_normalization/beta"]
        return W, b, gp, be

    def _inp(self, t, srcs, absolute=False):
        H = self.H[t]
        hu = self.plan.towers[t]["hidden"]
        parts = [self.X0 if s == "x" else H[s][:, :self.plan.out_width(hu[s])] for s in srcs]
        x = np.concatenate(parts, axis=1)
        return np.abs(x) if absolute else x

    def _tower_depth(self, t):
        return len(self.plan.towers[t]["hidden"])

    # ---- forward, per hidden layer
    def forward_checks(self):
        """Check of every hidden layer's output (criteria 1 and 2) and of its zero padding columns; the deep input's padding too."""
        out = []
        plan = self.plan
        pad = x0_padding_mask(plan)
        assert not np.any(self.X0p[:, pad]), "deep input: nonzero padding column"
        for t, tw in enumerate(plan.towers):
            hu, L = tw["hidden"], len(tw["hidden"])
            srcs = layer_sources(tw["mode"], L)
            for l in range(L):
                W, b, gp, be = self._layer_params(t, l, L)
                inp = self._inp(t, srcs[l])
                z = inp @ W + b
                a = act_fwd(self.act, z)
                keep = self._keep(t, l, a.shape[1])
                ad = a if keep is None else a * keep
                h = ad * gp + be if gp is not None else ad
                ks = 1.0 if keep is None else np.abs(keep)
                g_abs = 1.0 if gp is None else np.abs(gp)
                Mz = np.abs(inp) @ np.abs(W) + np.abs(b)
                Mh = g_abs * ks * LIP.get(self.act, 1.0) * Mz
                Rz = np.sqrt((inp * inp) @ (W * W))
                dact = np.abs(act_bwd_from_a(self.act, a)) if self.act in RELU_FAMILY else np.abs(_dz_from_z(self.act, z))
                Rh = g_abs * ks * dact * Rz
                slack = 2.0 ** -22 * (g_abs * np.abs(ad) + (0.0 if be is None else np.abs(be)))
                K = inp.shape[1] + 32
                gpu = self.H[t][l]
                n = h.shape[1]
                name = "tower %d layer %d (%s, %d units)" % (t, l, self.act, hu[l])
                assert not np.any(gpu[:, n:]), "%s: nonzero padding column" % name
                out.append(compare(name, gpu[:, :n], h, Mh, Rh, c_gemm(self.engine, K), slack))
        return out

    # ---- backward
    def head(self):
        """-> (logit, Mlogit, Rlogit2, Khead, wide): float64 logits from the GPU's last inputs, the same sum on absolute values, the
        sum of squared products, the longest fp32 accumulation of the head (wide ids + logits-layer inputs) and, per wide column,
        (column, example of each id, id)."""
        plan, B = self.plan, self.B
        logit, Mlogit, Rlogit2, Khead = np.zeros(B), np.zeros(B), np.zeros(B), 1
        wide = []
        if plan.use_wide:
            bias = self.params["linear/linear_model/bias_weights"][0]
            logit += bias
            Mlogit += abs(bias)
            for c in plan.wide_columns:
                rows, ids, cnt = self._col_ids(c)
                w = self.params["linear/linear_model/%s/weights" % c.name]
                np.add.at(logit, rows, w[ids])
                np.add.at(Mlogit, rows, np.abs(w[ids]))
                np.add.at(Rlogit2, rows, w[ids] ** 2)
                wide.append((c, rows, ids))
                Khead = max(Khead, int(cnt.max(initial=0)) * len(plan.wide_columns))
        for t, tw in enumerate(plan.towers):
            L = len(tw["hidden"])
            srcs = layer_sources(tw["mode"], L)
            W, b, _, _ = self._layer_params(t, L, L)
            inp = self._inp(t, srcs[L])
            logit += (inp @ W + b)[:, 0]
            Mlogit += (np.abs(inp) @ np.abs(W) + np.abs(b))[:, 0]
            Rlogit2 += ((inp * inp) @ (W * W))[:, 0]
            Khead += inp.shape[1]
        return logit, Mlogit, Rlogit2, Khead, wide

    def gradients(self):
        """-> (ref, M, R, C) dicts by tensor name: float64 gradients of every parameter the step touches, their magnitudes, the
        root-sum-squares of their last reduction (None where not a reduction) and the criterion-1 constant."""
        ref, M, R, Cd = {}, {}, {}, {}
        plan, B = self.plan, self.B
        w_abs = np.abs(self.weight)
        # logits from the GPU's last inputs (the head is an fp32 FFMA kernel: its error enters dlogit through sigmoid' <= 1/4)
        logit, Mlogit, Rlogit2, Khead, wide = self.head()
        sig = 1.0 / (1.0 + np.exp(-logit))
        dlogit = (sig - self.label) * self.weight
        Rd = sig * (1 - sig) * w_abs * np.sqrt(Rlogit2)          # (the head's products, through sigmoid')
        Kmax = max([B, Khead] + [self._inp(t, layer_sources(tw["mode"], len(tw["hidden"]))[l]).shape[1]
                                 for t, tw in enumerate(plan.towers) for l in range(len(tw["hidden"]) + 1)])
        depth = 2 + max([len(tw["hidden"]) + 1 for tw in plan.towers] or [0])
        C = c_gemm(self.engine, Kmax) * depth
        unc = 1.0 / C                                  # uncertainties that are not GEMM errors enter M scaled by 1 / C
        Md = np.abs(dlogit) + 0.25 * w_abs * (Khead + 2) * U * Mlogit * unc
        if plan.use_wide:
            ref["linear/linear_model/bias_weights"] = np.array([dlogit.sum()])
            M["linear/linear_model/bias_weights"] = np.array([Md.sum()])
            R["linear/linear_model/bias_weights"] = np.array([np.sqrt((dlogit ** 2 + Rd ** 2).sum())])
            for c, rows, ids in wide:
                name = "linear/linear_model/%s/weights" % c.name
                g, m, r = np.zeros(c.buckets), np.zeros(c.buckets), np.zeros(c.buckets)
                np.add.at(g, ids, dlogit[rows])
                np.add.at(m, ids, Md[rows])
                np.add.at(r, ids, dlogit[rows] ** 2 + Rd[rows] ** 2)
                ref[name], M[name], R[name] = g, m, np.sqrt(r)
        if plan.use_deep:
            dX, MdX, RdX = np.zeros_like(self.X0), np.zeros_like(self.X0), np.zeros_like(self.X0)
            for t in range(len(plan.towers)):
                self._tower_bwd(t, dlogit, Md, Rd, unc, dX, MdX, RdX, ref, M, R)
            for tb in plan.tables:
                name = "dnn/input_from_feature_columns/input_layer/%s/embedding_weights" % tb["name"]
                lo, po, w = plan.deep_layout[tb["name"]]
                rows, ids, cnt = self._col_ids(tb["column"])
                mw = self._bag_scale(cnt)[rows][:, None]
                g, m, r = (np.zeros((tb["rows"], tb["dim"])) for _ in range(3))
                np.add.at(g, ids, mw * dX[rows, lo:lo + w])
                np.add.at(m, ids, mw * MdX[rows, lo:lo + w])
                np.add.at(r, ids, mw ** 2 * (dX[rows, lo:lo + w] ** 2 + RdX[rows, lo:lo + w] ** 2))
                ref[name], M[name], R[name] = g, m, np.sqrt(r)
        for k in ref:
            Cd[k] = C
        self.dlogit = dlogit
        return ref, M, R, Cd

    def _tower_bwd(self, t, dlogit, Md, Rd, unc, dX, MdX, RdX, ref, M, R):
        plan, act = self.plan, self.act
        tw = plan.towers[t]
        hu, L = tw["hidden"], len(tw["hidden"])
        srcs = layer_sources(tw["mode"], L)
        dH = [np.zeros((self.B, plan.out_width(u))) for u in hu]
        MdH = [np.zeros_like(x) for x in dH]
        RdH = [np.zeros_like(x) for x in dH]          # (R of each data gradient, upstream operands' R included)

        def scatter(d, Md_, Rsq, sources):
            o = 0
            for s in sources:
                w = self.X0.shape[1] if s == "x" else plan.out_width(hu[s])
                g, m, r = (dX, MdX, RdX) if s == "x" else (dH[s], MdH[s], RdH[s])
                g += d[:, o:o + w]
                m += Md_[:, o:o + w]
                r[:] = np.sqrt(r ** 2 + Rsq[:, o:o + w])
                o += w

        W, _, _, _ = self._layer_params(t, L, L)
        inp = self._inp(t, srcs[L])
        sc = scope(t, L, L)
        ref[sc + "/kernel"] = inp.T @ dlogit[:, None]
        M[sc + "/kernel"] = np.abs(inp).T @ Md[:, None]
        d2 = dlogit ** 2 + Rd ** 2
        R[sc + "/kernel"] = np.sqrt((inp * inp).T @ d2[:, None])
        ref[sc + "/bias"], M[sc + "/bias"] = np.array([dlogit.sum()]), np.array([Md.sum()])
        R[sc + "/bias"] = np.array([np.sqrt(d2.sum())])
        scatter(dlogit[:, None] @ W.T, Md[:, None] @ np.abs(W).T, d2[:, None] @ (W * W).T, srcs[L])
        for l in range(L - 1, -1, -1):
            sc = scope(t, l, L)
            W, _, gp, be = self._layer_params(t, l, L)
            dh, Mdh, Rdh = dH[l], MdH[l], RdH[l]
            Hl = self.H[t][l][:, :dh.shape[1]]
            keep = self._keep(t, l, dh.shape[1])
            # post-activation value from H: a = (H - beta) / (gamma * inv), rounded to the fp32 value the kernels stored
            ad = Hl if gp is None else np.where(gp != 0, (Hl - be) / np.where(gp != 0, gp, 1.0), 0.0)
            if gp is not None or keep is not None:
                ad = ad.astype(np.float32).astype(np.float64)
            if keep is None:
                a = ad
            else:
                a = np.where(keep > 0, ad / np.where(keep > 0, keep, 1.0), 0.0).astype(np.float32).astype(np.float64)
                ad = a * keep
            if act == "relu6":                          # (H / (gamma * inv) of a clamped 6 may land an ulp below 6)
                a = np.where(np.abs(a - 6) <= 8 * ulp32(6.0), 6.0, a)
            if gp is not None:
                ref[sc + "/batch_normalization/gamma"] = (dh * ad).sum(0) * GAMMA_SCALE
                M[sc + "/batch_normalization/gamma"] = (Mdh * np.abs(ad)).sum(0) * GAMMA_SCALE
                R[sc + "/batch_normalization/gamma"] = np.sqrt(((dh ** 2 + Rdh ** 2) * ad ** 2).sum(0)) * GAMMA_SCALE
                ref[sc + "/batch_normalization/beta"] = dh.sum(0)
                M[sc + "/batch_normalization/beta"] = Mdh.sum(0)
                R[sc + "/batch_normalization/beta"] = np.sqrt((dh ** 2 + Rdh ** 2).sum(0))
                da, Mda, Rda = dh * gp, Mdh * np.abs(gp), Rdh * np.abs(gp)
            else:
                da, Mda, Rda = dh, Mdh, Rdh
            if keep is not None:
                da, Mda, Rda = da * keep, Mda * keep, Rda * keep
            d1 = act_bwd_from_a(act, a)
            # act' from the stored a: a may sit an ulp away from the kernels' a, and act_bwd itself rounds in fp32
            d1_unc = 0.0 if act in RELU_FAMILY else (DLIP[act] * 2 * ulp32(a) + 2.0 ** -22) * unc
            if act == "crelu":
                u = dh.shape[1] // 2
                dz = da[:, :u] * d1[:, :u] - da[:, u:] * d1[:, u:]
                Mdz = Mda[:, :u] * d1[:, :u] + Mda[:, u:] * d1[:, u:]
                Rdz = np.sqrt((Rda[:, :u] * d1[:, :u]) ** 2 + (Rda[:, u:] * d1[:, u:]) ** 2)
                W = W[:, :u]
            else:
                dz = da * d1
                Mdz = Mda * (np.abs(d1) + d1_unc)
                Rdz = Rda * np.abs(d1)
            z2 = dz * dz + Rdz * Rdz
            inp = self._inp(t, srcs[l])
            ref[sc + "/kernel"] = inp.T @ dz
            M[sc + "/kernel"] = np.abs(inp).T @ Mdz
            R[sc + "/kernel"] = np.sqrt((inp * inp).T @ z2)
            ref[sc + "/bias"], M[sc + "/bias"] = dz.sum(0), Mdz.sum(0)
            R[sc + "/bias"] = np.sqrt(z2.sum(0))
            scatter(dz @ W.T, Mdz @ np.abs(W).T, z2 @ (W * W).T, srcs[l])

    def gradient_checks(self, grads, before, names=None):
        """Criteria 1 and 2 for every gradient the step produced (grads, before: probe_step's result and the uploaded params)."""
        ref, M, R, C = self.gradients()
        out = []
        for name in (names or ref):
            g = grads[name].reshape(ref[name].shape)
            slack = 2.0 ** -47 * np.abs(before[name].astype(np.float64)).reshape(ref[name].shape)    # SGD read-back rounding
            # criterion 2 is for the dense layers' GEMM and batch reductions: an embedding or wide row sums a handful of dX0 or dlogit
            # values, whose error is the head's and the data gradients', not a reduction of its own
            dense = name.startswith("dnn/dnn_")
            out.append(compare(name, g, ref[name], M[name], R[name] if dense else None, C[name], slack))
        # parameters the step cannot touch (untouched embedding / wide rows) come back exactly unchanged
        for name in grads:
            if name not in ref:
                assert not np.any(grads[name]), "%s: gradient where the reference has none" % name
        return out


# ------------------------------------------------------------------------------------------------ configurations and batches
SGD_PROBE = "tf.train.GradientDescentOptimizer(learning_rate=16777216.0)"


def parity_conf(hidden, mode="simple", act="relu", bn=1, dropout=0.0, opt=SGD_PROBE):
    """Three hashed columns (c2 hot: few buckets; tags multihot) and two numeric ones, one with a bucketized wide twin.  With
    embedding_dim_override 8 the deep input is 26 wide (d0_phys 32); with 64 it is 197 wide (d0_phys 224)."""
    from collections import OrderedDict
    fc = OrderedDict()
    fc["c1"] = dict(type="category", transform="hash_bucket", parameter=3000)
    fc["c2"] = dict(type="category", transform="hash_bucket", parameter=40)
    fc["tags"] = dict(type="category", transform="hash_bucket", parameter=5000)
    fc["x1"] = dict(type="continuous", transform=None, parameter=dict(normalization=None, boundaries=None))
    fc["x2"] = dict(type="continuous", transform="standard", parameter=dict(normalization=[0.0, 2.0], boundaries=[-1, 0, 1]))
    model = dict(linear_optimizer=opt, linear_initial_learning_rate=0.05, dnn_hidden_units=[list(h) for h in hidden] if
                 isinstance(hidden[0], (list, tuple)) else list(hidden), dnn_connected_mode=mode, dnn_optimizer=opt,
                 dnn_initial_learning_rate=0.05, dnn_activation_function=act, dnn_dropout=dropout or None, dnn_batch_normalization=bn)
    return fc, [], model


def raw_batch(B, rng, dense_scale=1.0):
    """Raw batch (oracle format) for parity_conf: c1 uniform over 2000 tokens, c2 over 60, tags 0-24 Zipf ids per row (hot rows
    get far more than 16 occurrences in a batch), x1 ~ N(0, dense_scale), x2 ~ N(0, 2)."""
    from oracle import hashing as OH
    raw = {}
    for f, n in (("c1", 2000), ("c2", 60)):
        offs = np.arange(B + 1, dtype=np.int64)
        raw[f] = (offs, OH.fingerprint64_tokens(["%s_%d" % (f, i) for i in rng.integers(0, n, size=B)]))
    lens = np.clip(rng.poisson(6, size=B), 0, 24)
    offs = np.zeros(B + 1, dtype=np.int64)
    offs[1:] = np.cumsum(lens)
    ids = (rng.zipf(1.3, size=int(offs[-1])) - 1) % 800
    raw["tags"] = (offs, OH.fingerprint64_tokens(["t%d" % i for i in ids]))
    raw["x1"] = (rng.standard_normal(B) * dense_scale).astype(np.float32)
    raw["x2"] = (rng.standard_normal(B) * 2).astype(np.float32)
    return raw


def random_params(names_shapes, rng, act):
    """fp32 parameters for a probe: glorot-scale kernels, small biases, gamma in [0.5, 1.5], beta 0 for relu-family gates (the
    sign of a = H / (gamma * inv) is then exact) and small random beta for smooth activations; embeddings ~ N(0, 0.3), wide
    weights ~ N(0, 0.1)."""
    out = {}
    for name, shape in names_shapes:
        if name.endswith("/kernel"):
            v = rng.uniform(-1, 1, size=shape) * np.sqrt(6.0 / (shape[0] + shape[1]))
        elif name.endswith("/gamma"):
            v = rng.uniform(0.5, 1.5, size=shape)
        elif name.endswith("/beta"):
            v = np.zeros(shape) if act in RELU_FAMILY else rng.uniform(-0.3, 0.3, size=shape)
        elif name.endswith("/bias") and name.startswith("dnn/"):
            v = rng.uniform(-0.1, 0.1, size=shape)
        elif "embedding_weights" in name:
            v = rng.standard_normal(shape) * 0.3
        else:
            v = rng.standard_normal(shape) * 0.1
        out[name] = np.ascontiguousarray(v, dtype=np.float32)
    return out


def _dz_from_z(name, z):
    """d act / d z from z (float64), for the RMS weight of smooth activations in the forward check."""
    from oracle.model import act_bwd
    return act_bwd(name, z, act_fwd(name, z))
