"""fp64 reference of the fused local-attention op and of block_extractor, with the error magnitudes that bound what a
16-bit kernel may return.

The reference follows the kernels' tap selection bit for bit (axis_tap in csrc/common.cuh: d = (flow + offset) + coord
in the arithmetic type A -- fp32, or fp64 for fp64 data (Acc<double>, common.cuh:18-19) --, floor, clamp, weights 1 - frac
and frac in A) and does everything else in fp64: softmax of the logits as
stored, the literal 4 k^2 bilinear corners of every pixel summed into one sparse matrix W[pixel, source position] per
image (1/k^2 included; duplicate corners are the border fold), and sparse algebra on that.

Next to each value it returns the magnitudes a rounding analysis needs (sums of absolute values of the terms that make
it up), and the bound_* functions turn them into a per-element bound |y - ref| <= bound for a given unit roundoff u and
absolute floor eta.  assert_within checks a kernel output against one.  See DESIGN.md section 6.
"""
import numpy as np
import scipy.sparse as sps

# unit roundoff of round-to-nearest storage: 8 significant bits (bf16), 11 (fp16)
U_BF16, U_FP16 = 2.0 ** -8, 2.0 ** -11
# absolute floor: half the subnormal spacing of the storage type (bf16 shares fp32's range, so it never matters)
ETA_BF16, ETA_FP16 = 2.0 ** -133, 2.0 ** -25
GW, GH = 16, 8          # tile kernels' pixel group, row-major per image (tile_window.cuh:12-25)

# fp32 arithmetic around a 16-bit rounding in the tile kernels (k = 3, 5): softmax (pixel_softmax,
# local_attn_pixel.cuh:19-35), the window weights (build_window, tile_window.cuh:77-92) and at most (k+1)^2 = 36 products
# per output summed in the MMA accumulators (local_attn_tc.cu:150): a few dozen fp32 roundings, each <= 2^-24 of the
# magnitude.  The CUDA-core gather kernels take their fp32 term from ref64_gather instead, which grows with k and C.
FP32_SLACK = 2.0 ** -20


def storage(name):
    """-> (u, eta) of a 16-bit storage type ('bf16' or 'fp16')"""
    return {"bf16": (U_BF16, ETA_BF16), "fp16": (U_FP16, ETA_FP16)}[name]


def gamma(n):
    """headroom for n fp32 products summed in fp32: 4 n 2^-24.  The tensor cores' fp32 accumulation (local_attn_bwd_tc.cu:
    48-53, the P GEMM behind Q) is not guaranteed to round to nearest, hence 4x the sequential-sum bound n 2^-24."""
    return n * 2.0 ** -22


def round_bf16(x):
    """round to nearest even bf16 (through fp32, as __float2bfloat16_rn of an fp32 value), returned as fp64"""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(np.float32).astype(np.float64)


def round_fp16(x):
    return np.asarray(np.asarray(x, np.float32), np.float16).astype(np.float64)


def axis_taps(flow, k, coord, dim, A=np.float32):
    """The k taps along one axis, exactly as axis_tap (common.cuh:51-62) in the arithmetic type A (np.float32 or
    np.float64): flow (any shape, converted to A), coord broadcastable.
    -> lo, hi, fl (int64) and wlo, whi (fp64 copies of the A weights), each of shape (k,) + flow.shape"""
    f = np.asarray(flow, A)
    off = (np.arange(k) - k // 2).astype(A).reshape((k,) + (1,) * f.ndim)
    d = (f[None] + off) + np.asarray(coord, A)[None]                 # A + A, rounded after each add
    fd = np.floor(d)
    fl = fd.astype(np.int64)
    lo = np.clip(fl, 0, dim - 1)
    hi = np.clip((fd + A(1)).astype(np.int64), 0, dim - 1)
    frac = d - fd                                                     # exact
    wlo = A(1) - frac                                                 # one rounding in A, as in the kernel
    return lo, hi, fl, wlo.astype(np.float64), frac.astype(np.float64)


class Taps:
    """Per-pixel taps of a flow field [B, 2, H, W] over a source of Hs x Ws, selected in the arithmetic type A (16-bit
    flows are widened to fp32 first, as ld() does).  Corner c of tap (i, j) of pixel n: position pos[b, i, j, c, n],
    bilinear weight cw[b, i, j, c, n]; corners in the order LT, RT, LB, RB of tap_value (local_attn_pixel.cuh:55-62)."""

    def __init__(self, flow, k, Hs, Ws, A=np.float32):
        flow = np.asarray(flow, A)
        self.B, _, self.H, self.W = flow.shape
        self.k, self.Hs, self.Ws, self.A = k, Hs, Ws, A
        ys, xs = np.meshgrid(np.arange(self.H), np.arange(self.W), indexing="ij")
        self.ty = axis_taps(flow[:, 1], k, ys[None], Hs, A)  # each (k, B, H, W)
        self.tx = axis_taps(flow[:, 0], k, xs[None], Ws, A)
        self.build()

    def build(self):
        """(re)derive corner positions and weights from self.tx / self.ty (tests edit those to inject faults)"""
        k, B, N = self.k, self.B, self.H * self.W
        ylo, yhi, yfl, ywlo, ywhi = (a.reshape(k, B, N) for a in self.ty)
        xlo, xhi, xfl, xwlo, xwhi = (a.reshape(k, B, N) for a in self.tx)
        steps = np.arange(k).reshape(k, 1, 1)
        self.regular = (np.all(yfl == yfl[:1] + steps, axis=0) & np.all(xfl == xfl[:1] + steps, axis=0))   # (B, N)
        Y = np.stack([ylo, ylo, yhi, yhi], 1)[:, None]        # (k_i, 1, 4, B, N)
        X = np.stack([xlo, xhi, xlo, xhi], 1)[None]           # (1, k_j, 4, B, N)
        WY = np.stack([ywlo, ywlo, ywhi, ywhi], 1)[:, None]
        WX = np.stack([xwlo, xwhi, xwlo, xwhi], 1)[None]
        self.pos = np.moveaxis(Y * self.Ws + X, 3, 0)         # (B, k, k, 4, N)
        self.cw = np.moveaxis(WY * WX, 3, 0)
        self.wx = (xwlo, xwhi)                                # per-axis weights for the flow gradient, (k, B, N)
        self.wy = (ywlo, ywhi)


def softmax64(logits):
    lg = np.asarray(logits, np.float64)
    e = np.exp(lg - lg.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


def _cl(a, b):
    """image b of [B, C, h, w] as a channels-last (h w, C) fp64 matrix"""
    return np.ascontiguousarray(np.asarray(a[b], np.float64).reshape(a.shape[1], -1).T)


class LocalAttn:
    """fp64 reference of out[b, c, y, x] = 1/k^2 sum_t softmax(logits)[t] bilinear_t(source[b, c]) and its gradients,
    with the taps of a kernel that computes in A."""

    def __init__(self, flow, logits, k, Hs, Ws, A=np.float32):
        self.taps = Taps(flow, k, Hs, Ws, A)
        self.k = k
        self.p = softmax64(logits)                            # (B, k^2, H, W)
        self.build()

    def build(self):
        t = self.taps
        B, k, N = t.B, self.k, t.H * t.W
        pr = self.p.reshape(B, k, k, 1, N) / (k * k)
        self.wts = pr * t.cw                                  # (B, k, k, 4, N): p_t / k^2 * bilinear corner weight
        rows = np.broadcast_to(np.arange(N), t.pos.shape[1:])
        self.W = [sps.csr_matrix((self.wts[b].ravel(), (rows.ravel(), t.pos[b].ravel())), shape=(N, t.Hs * t.Ws))
                  for b in range(B)]                          # duplicates summed = the border fold

    def _apply(self, mats, a, shape, chunk=64):
        B, C = a.shape[:2]
        out = np.empty((B, C) + shape)
        for b in range(B):
            for c0 in range(0, C, chunk):
                blk = np.asarray(a[b, c0:c0 + chunk], np.float64).reshape(min(chunk, C - c0), -1)
                out[b, c0:c0 + chunk] = (mats[b] @ blk.T).T.reshape((-1,) + shape)
        return out

    def fwd(self, src):
        """-> out, M = W |S|"""
        t = self.taps
        src = np.asarray(src, np.float64)
        return self._apply(self.W, src, (t.H, t.W)), self._apply(self.W, np.abs(src), (t.H, t.W))

    def probs(self):
        return self.p

    def bwd(self, src, gout):
        """-> dict: gs = W^T G, Mgs = W^T |G|; per tap q / qa (corner dot products g.s and |g|.|s|, (B, k, k, 4, N)),
        dp, D (the same formula with qa), PD = sum_u p_u D_u; gl, gf (x plane, then y), Mgf; n_adds"""
        t, k = self.taps, self.k
        B, N, KK = t.B, t.H * t.W, k * k
        src = np.asarray(src, np.float64)
        gout = np.asarray(gout, np.float64)
        WT = [w.T.tocsr() for w in self.W]
        gs = self._apply(WT, gout, (t.Hs, t.Ws))
        Mgs = self._apply(WT, np.abs(gout), (t.Hs, t.Ws))
        q = np.empty(t.pos.shape)
        qa = np.empty(t.pos.shape)
        for b in range(B):
            S, G = _cl(src, b), _cl(gout, b)
            aS, aG = np.abs(S), np.abs(G)
            for i in range(k):
                for j in range(k):
                    for c in range(4):
                        ps = t.pos[b, i, j, c]
                        q[b, i, j, c] = np.einsum("nc,nc->n", G, S[ps])
                        qa[b, i, j, c] = np.einsum("nc,nc->n", aG, aS[ps])
        r = self.grads_from_q(q)
        p = self.p.reshape(B, KK, N)
        D = (t.cw * qa).sum(axis=3).reshape(B, KK, N) / KK
        r["D"] = D.reshape(self.p.shape)
        r["PD"] = (p * D).sum(axis=1).reshape(B, 1, t.H, t.W)
        r["Mgf"] = self.flow_mag(qa, self.p.reshape(B, k, k, N) / KK)
        r.update(gs=gs, Mgs=Mgs, q=q, qa=qa, n_adds=self.n_adds())
        return r

    def flow_mag(self, qa, pw):
        """tap_backward's grad_flow terms with |g|.|s| for the dot products (the error of a dot product scales with that,
        not with its value), each tap's weighted by pw (B, k, k, N) in place of p / k^2.  -> (B, 2, H, W), x plane first"""
        t = self.taps
        (xwlo, xwhi), (ywlo, ywhi) = t.wx, t.wy
        mx = pw * (ywlo.transpose(1, 0, 2)[:, :, None] * (qa[:, :, :, 0] + qa[:, :, :, 1])
                   + ywhi.transpose(1, 0, 2)[:, :, None] * (qa[:, :, :, 2] + qa[:, :, :, 3]))
        my = pw * (xwlo.transpose(1, 0, 2)[:, None] * (qa[:, :, :, 0] + qa[:, :, :, 2])
                   + xwhi.transpose(1, 0, 2)[:, None] * (qa[:, :, :, 1] + qa[:, :, :, 3]))
        return np.stack([mx.sum(axis=(1, 2)), my.sum(axis=(1, 2))], 1).reshape(t.B, 2, t.H, t.W)

    def grads_from_q(self, q):
        """dp, grad_logits and grad_flow from the corner dot products (tap_backward / store_pixel_grads, fp64)"""
        t, k = self.taps, self.k
        B, N, KK = t.B, t.H * t.W, k * k
        dp = (t.cw * q).sum(axis=3).reshape(B, KK, N) / KK
        p = self.p.reshape(B, KK, N)
        gl = p * (dp - (p * dp).sum(axis=1, keepdims=True))
        pij = self.p.reshape(B, k, k, N) / KK
        (xwlo, xwhi), (ywlo, ywhi) = t.wx, t.wy
        xl, xh = xwlo.transpose(1, 0, 2)[:, None], xwhi.transpose(1, 0, 2)[:, None]      # (B, 1, k_j, N)
        yl, yh = ywlo.transpose(1, 0, 2)[:, :, None], ywhi.transpose(1, 0, 2)[:, :, None]  # (B, k_i, 1, N)
        qLT, qRT, qLB, qRB = (q[:, :, :, c] for c in range(4))
        gfy = (pij * (-xl * qLT - xh * qRT + xl * qLB + xh * qRB)).sum(axis=(1, 2))
        gfx = (pij * (-yl * qLT - yh * qLB + yl * qRT + yh * qRB)).sum(axis=(1, 2))
        return {"dp": dp.reshape(self.p.shape), "gl": gl.reshape(self.p.shape),
                "gf": np.stack([gfx, gfy], 1).reshape(B, 2, t.H, t.W)}

    def n_adds(self):
        """bf16 roundings of the running sum of one grad_source element in the tile backward, per image position
        (B, Hs, Ws): inside the image one bf16 atomic add per 16x8 pixel group with a non-zero window entry there
        (local_attn_bwd_tc.cu, the bf16x2 atomicAdd of the GS epilogue); on the border the groups' adds are summed in fp32
        and rounded once (k_fold_border).  Plus one per corner tap of an irregular pixel there (irregular_pixel_bwd's
        red_add)."""
        t = self.taps
        N, gcols = t.H * t.W, (t.W + GW - 1) // GW
        ys, xs = np.divmod(np.arange(N), t.W)
        gid = (ys // GH) * gcols + xs // GW
        ngroups = int(gid.max()) + 1
        out = np.zeros((t.B, t.Hs * t.Ws))
        border = border_mask(t.Hs, t.Ws).ravel()
        for b in range(t.B):
            reg = t.regular[b]
            nz = sps.diags(reg.astype(np.float64)) @ (self.W[b] != 0).astype(np.float64)
            grp = sps.csr_matrix((np.ones(N), (gid, np.arange(N))), shape=(ngroups, N))
            out[b] = np.asarray(((grp @ nz) > 0).sum(axis=0)).ravel()
            out[b][border] = 1.0
            out[b] += np.bincount(t.pos[b][:, :, :, ~reg].ravel(), minlength=t.Hs * t.Ws)
        return out.reshape(t.B, t.Hs, t.Ws)


def border_mask(Hs, Ws):
    """source positions on the image border (rows 0 and Hs-1, columns 0 and Ws-1)"""
    m = np.zeros((Hs, Ws), bool)
    m[[0, -1], :] = True
    m[:, [0, -1]] = True
    return m


def block_extract(src, flow, k, gout=None, A=np.float32):
    """fp64 block_extractor with the taps of a kernel that computes in A: out [B, C, k H, k W] (out[.., y k + i, x k + j]
    = bilinear tap (i, j) of pixel (y, x)) and its magnitude; with gout also grad_source, grad_flow and their magnitudes,
    and "taps" (the Taps)."""
    src = np.asarray(src, np.float64)
    B, C, Hs, Ws = src.shape
    t = Taps(flow, k, Hs, Ws, A)
    H, W, N = t.H, t.W, t.H * t.W
    r = {"out": np.empty((B, C, H, k, W, k)), "M": np.empty((B, C, H, k, W, k)), "taps": t}
    if gout is not None:
        g6 = np.asarray(gout, np.float64).reshape(B, C, H, k, W, k)
        for key, shp in (("gs", (B, Hs * Ws, C)), ("Mgs", (B, Hs * Ws, C)), ("gf", (B, 2, N)), ("Mgf", (B, 2, N))):
            r[key] = np.zeros(shp)
    (xwlo, xwhi), (ywlo, ywhi) = t.wx, t.wy
    for b in range(B):
        S = _cl(src, b)
        for i in range(k):
            for j in range(k):
                v = [S[t.pos[b, i, j, c]] for c in range(4)]                   # (N, C) each
                w = [t.cw[b, i, j, c][:, None] for c in range(4)]
                r["out"][b, :, :, i, :, j] = sum(w[c] * v[c] for c in range(4)).T.reshape(C, H, W)
                r["M"][b, :, :, i, :, j] = sum(w[c] * np.abs(v[c]) for c in range(4)).T.reshape(C, H, W)
                if gout is None:
                    continue
                g = g6[b, :, :, i, :, j].reshape(C, N).T                       # (N, C)
                for c in range(4):
                    np.add.at(r["gs"][b], t.pos[b, i, j, c], w[c] * g)
                    np.add.at(r["Mgs"][b], t.pos[b, i, j, c], w[c] * np.abs(g))
                xl, xh = xwlo[j, b][:, None], xwhi[j, b][:, None]
                yl, yh = ywlo[i, b][:, None], ywhi[i, b][:, None]
                r["gf"][b, 1] += (g * (-xl * v[0] - xh * v[1] + xl * v[2] + xh * v[3])).sum(1)
                r["gf"][b, 0] += (g * (-yl * v[0] - yh * v[2] + yl * v[1] + yh * v[3])).sum(1)
                ag = np.abs(g)
                r["Mgf"][b, 1] += (ag * (xl * (np.abs(v[0]) + np.abs(v[2])) + xh * (np.abs(v[1]) + np.abs(v[3])))).sum(1)
                r["Mgf"][b, 0] += (ag * (yl * (np.abs(v[0]) + np.abs(v[1])) + yh * (np.abs(v[2]) + np.abs(v[3])))).sum(1)
    r["out"] = r["out"].reshape(B, C, k * H, k * W)
    r["M"] = r["M"].reshape(B, C, k * H, k * W)
    if gout is not None:
        r["gs"] = r["gs"].transpose(0, 2, 1).reshape(B, C, Hs, Ws)
        r["Mgs"] = r["Mgs"].transpose(0, 2, 1).reshape(B, C, Hs, Ws)
        r["gf"] = r["gf"].reshape(B, 2, H, W)
        r["Mgf"] = r["Mgf"].reshape(B, 2, H, W)
    return r


# ----------------------------------------------------------------------------------------------------------- bounds
# Each returns the per-element bound on |y - ref|.  u, eta: storage(...).  init: what an accumulate=1 call's buffer held.

def bound_out_tile(r, M, u, eta):
    """tile forward (local_attn_tc.cu): bf16 window (build_window's bf16 pack, tile_window.cuh:120: <= u of each weight,
    so u M), fp32 accumulation (FP32_SLACK M), one bf16 store (local_attn_tc.cu:183-186: u |r + error|, the 1.01 pays
    for u of the error terms)"""
    return 1.01 * u * (np.abs(r) + M) + FP32_SLACK * M + eta


def bound_gather16(r, e32, u, eta):
    """any output of the CUDA-core kernels (gather local attention, block_extractor) in 16-bit storage: the fp32 kernel's
    arithmetic on the widened values -- e32, its ref64_gather bound -- and one rounding to the storage type (st(), the
    narrowing of the fp32 grad_source buffer in functional.block_extract_bwd, or of the fp32 copies' gradients in
    functional.local_attn_bwd): u |r + err| <= u (|r| + e32)"""
    return u * np.abs(r) + (1 + u) * e32 + eta


def blend_ref(r, M, prev, mask):
    """out = prev (1 - m) + attn m: reference and magnitude (local_attn.cu:96, local_attn_tc.cu:179-180); the fp32 blend
    adds its own roundings of the prev term, so |prev| (1 - m) joins the magnitude"""
    return prev * (1 - mask) + r * mask, M * mask + np.abs(prev) * (1 - mask)


def bound_out_tile_blend(r, M, Mattn, u, eta):
    """tile forward with blend: the bf16 window rounding scales with the attention part only (Mattn = m W|S|); M =
    blend_ref's magnitude"""
    return 1.01 * u * (np.abs(r) + Mattn) + FP32_SLACK * M + eta


def bound_probs(p, u, eta):
    """softmax in fp32 (pixel_softmax, FP32_SLACK absolute, p <= 1), one 16-bit store (local_attn_tc.cu:94, u p)"""
    return u * p + FP32_SLACK + eta


def bound_gs_tile(Mgs, n_adds, u, eta, init=0.0):
    """tile backward grad_source: per element n_adds roundings of the running sum (<= Mgs + |init|): bf16 atomic adds,
    or on the border the one rounding of k_fold_border (LocalAttn.n_adds); + 2 for the bf16 window (tile_window.cuh:120,
    u Mgs) and the bf16 rounding of each group's partial (__floats2bfloat162_rn in the GS epilogue of
    local_attn_bwd_tc.cu, u Mgs in total); fp32 MMA accumulation of the partials (FP32_SLACK Mgs)"""
    return u * (n_adds + 2) * (Mgs + np.abs(init)) + FP32_SLACK * Mgs + eta


def bound_gl(r, p, D, PD, C, u, eta, init=0.0):
    """grad_logits = p_t (dp_t - sum_u p_u dp_u): every dot product over C channels carries gamma(C) of its |g|.|s| sum,
    so dp_t carries gamma(C) D_t (tap_backward, local_attn_pixel.cuh:69); one 16-bit store (store_pixel_grads,
    local_attn_pixel.cuh:86, u |r|); the fp32 add of the buffer's initial value (same line, FP32_SLACK |init|)"""
    return u * np.abs(r) + gamma(C) * p * (D + PD) + FP32_SLACK * np.abs(init) + eta


def bound_gf(r, Mgf, C, u=0.0, eta=0.0, init=0.0):
    """grad_flow: gamma(C) of the dot products through tap_backward's flow sums (local_attn_pixel.cuh:70-71, Mgf); the
    fp32 sum over the taps and the add of the initial value (local_attn_pixel.cuh:88-89, FP32_SLACK); with a 16-bit flow
    one store in that type (u |r| + eta)"""
    return gamma(C) * Mgf + FP32_SLACK * (np.abs(r) + np.abs(init)) + u * np.abs(r) + eta


def bound_be_gf(r, mag, n, u=0.0, eta=0.0):
    """block_extractor grad_flow with every flow element owned by one thread (the deterministic backward's single channel
    slice): n = k^2 C products summed in fp32 per flow element (block_extract.cu:96-105, gamma(n) mag), with a 16-bit
    flow one store in that type (u |r| + eta)"""
    return gamma(n) * mag + u * np.abs(r) + eta


# ------------------------------------------------------------------------------------------------------- assertion
def check(name, y, ref, bound, **mags):
    """-> (max |y - ref| / bound, message); message is None when every element is within its bound"""
    y = np.asarray(y, np.float64)
    ref = np.asarray(ref, np.float64)
    bound = np.broadcast_to(np.asarray(bound, np.float64), ref.shape)
    ratio = np.abs(y - ref) / bound
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    worst = float(ratio.max())
    if worst <= 1.0:
        return worst, None
    idx = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    parts = [f"{name}: {int((ratio > 1).sum())} of {ratio.size} elements exceed their bound; worst |err|/bound = "
             f"{worst:.3g} at {tuple(int(i) for i in idx)}: y = {y[idx]!r}, ref = {ref[idx]!r}, bound = {bound[idx]!r}"]
    for k, v in mags.items():
        parts.append(f"{k} = {np.broadcast_to(np.asarray(v, np.float64), ref.shape)[idx]!r}")
    return worst, ", ".join(parts)


def assert_within(name, y, ref, bound, **mags):
    """assert |y - ref| <= bound element-wise; on failure report the worst ratio, its index, the reference and the
    magnitudes there, and how many elements fail.  Returns the worst ratio."""
    worst, msg = check(name, y, ref, bound, **mags)
    assert msg is None, msg
    return worst
