"""Float64 reference of the tracker's per-level sums (calcRes + calcGSSSE), with a derived error bound for each output.

The per-point inputs come from the oracle, which is pinned bit for bit to the reference: `orc.CoarseTracker.calcRes` followed by
`warped()` gives {idepth, u, v, dx, dy, residual, hw, refColor} of every point that lands in buf_warped_* (in bounds, finite, not
saturated), and `rs` gives nE and nSat.  From those the module forms every point's terms in float32 with the kernels' expression trees
(`eval_point` / `stage_accumulate` / `flow_point`, compiled with --fmad=false, so numpy's IEEE float32 operations reproduce them):

  * J[0..8], Jw = J*hw rounded to float32, and the outer-product term Jw_r*J_c rounded once to float32 (what fmaf(Jw, J, 0) gives);
  * the energy e_i = hw*r*r*(2-hw) of every warped point and maxEnergy for every saturated one;
  * the flow indicators of every level-0 point with i % 32 == 0, with RKi, t and Ki exactly as make_eval_params builds them.

Each output entry is then summed exactly (math.fsum) and A = sum |t_i| is recorded, and the kernels' finalisation is applied:
finalize_res (float casts of E, nE, nSat and the flow sums) and finalize_gs (float cast, 1.0f/npad over the padded count, SCALE_*).

Error bound.  Let u = 2^-24 (unit roundoff of float32).  A kernel in which every thread adds at most m terms into one float32 accumulator
and then hands the partial to fp64 reductions computes, for an output entry with exact sum S of reference terms and absolute sum A:
  * the per-thread recursive float sum of m terms starting from 0: |error| <= (m-1) u sum|t| (first order; gamma_{m-1} < 1.001 (m-1) u here);
  * for H/b the terms are fmaf products, exact before the add: each product that the reference rounds once differs from the exact product
    by at most u|t|, one more u A in total, so (m+1) u A covers H, b and E (E's terms are the same float32 numbers on both sides);
  * the fp64 block / cluster / grid reductions add at most (#adds) 2^-53 A, under 1e-12 A for any launch here;
  * finalisation rounds the fp64 total to float32, and the reference rounds S the same way: |fl(x) - fl(S)| <= |x - S| + u|x| + u|S|,
    i.e. 2 u |S| more (to first order);
  * then the same exact scale factors (1.0f/npad, SCALE_*) multiply both sides in double.
So  bound(m) = (1.001 (m+1) u A + 1e-12 A + 2 u |S|) * |scale|.  The flow sums add two terms per flow point, so they use 2m in place of m.
lastResiduals = sqrtf((float)(E/nE)) adds two float roundings: |d lr| <= lr (bound_E / 2E + 2u).

m comes from the launch geometry: the step-wise kernel runs G = min(ceil(n/256), 4 SMs) blocks of 256 threads, m = ceil(n/(256 G));
the LM kernel runs one cluster of C CTAs of THREADS threads per job, m = ceil(n/(THREADS C)).  The oracle itself sums E and the flow
in ONE float (m = number of terms) and H/b in 4 SSE lanes with 1000-term tiers (m = ceil(npad/4) plus one rounding per tier shift and
the 3 lane adds).
"""
import math
import numpy as np

F = np.float32
U = 2.0 ** -24
SC = [1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 10.0, 1000.0]            # SCALE_XI_ROT x3, SCALE_XI_TRANS x3, SCALE_A, SCALE_B
RC = [(r, c) for r in range(9) for c in range(r, 9)]           # row-major upper triangle of the 9x9 system (45 entries)
IDX_E, IDX_FT, IDX_FRT = 45, 46, 47                            # entries of Ref.S / Ref.A after the 45 system entries


def m_step(n, sms):
    """Points per thread of the step-wise kernel (coarse_res_gs_kernel, 256 threads, grid capped at 4 blocks per SM)."""
    if n <= 0:
        return 0
    G = min(-(-n // 256), 4 * sms)
    return -(-n // (256 * G))


def m_lm(n, threads, cluster):
    """Points per thread of track_cluster_kernel (one cluster of `cluster` CTAs per job)."""
    return -(-n // (threads * cluster)) if n > 0 else 0


def m_oracle_gs(npad):
    """Accumulator9: 4 lanes, 1000-update tiers, 3 lane adds at finish."""
    q = -(-npad // 4)
    return q + 2 * (-(-q // 1000)) + 5


def qmat(q):
    """Quaternion {w,x,y,z} -> row-major rotation, double, the expression of sdv_math.cuh / Eigen toRotationMatrix."""
    w, x, y, z = (float(v) for v in q)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]]


def eval_params(T7, Ki, a, b, ref_a=0.0, ref_b=0.0, ref_exposure=1.0, new_exposure=1.0):
    """make_eval_params: RKi (float32, from the double rotation cast to float), t (float32), aLL, bLL, b0."""
    R = qmat(T7[:4]); Rf = [[F(v) for v in row] for row in R]; Ki = np.asarray(Ki, F)
    RKi = np.array([[(Rf[i][0] * Ki[0, j] + Rf[i][1] * Ki[1, j]) + Rf[i][2] * Ki[2, j] for j in range(3)] for i in range(3)], F)
    t = np.array([F(T7[4]), F(T7[5]), F(T7[6])], F)
    eF, eT = float(F(ref_exposure)), float(F(new_exposure))
    if eF == 0 or eT == 0:
        eF = eT = 1.0
    al = math.exp(a - ref_a) * eT / eF
    return RKi, t, F(al), F(b - al * ref_b), F(ref_b)


def _fsum(x):
    return math.fsum(np.asarray(x, np.float64).tolist())


def flow_terms(cloud, K4, Ki, RKi, t):
    """Float32 flow-indicator terms of the points with i % 32 == 0 (flow_point / CoarseTracker.cpp:538-566), in the order the kernels add them."""
    x, y, idp = (np.asarray(c, F)[::32] for c in cloud[:3])
    fx, fy, cx, cy = (F(v) for v in K4); one = F(1)
    Ki = np.asarray(Ki, F)

    def proj(M, sgn):
        p = [((M[i, 0] * x + M[i, 1] * y) + M[i, 2] * one) + sgn * (t[i] * idp) for i in range(3)]
        return fx * (p[0] / p[2]) + cx, fy * (p[1] / p[2]) + cy

    def sq(Ku, Kv):
        return (Ku - x) * (Ku - x) + (Kv - y) * (Kv - y)

    with np.errstate(all="ignore"):
        tT = np.stack([sq(*proj(Ki, F(1))), sq(*proj(Ki, F(-1)))], 1).reshape(-1)
        tRT = np.stack([sq(*proj(RKi, F(1))), sq(*proj(RKi, F(-1)))], 1).reshape(-1)
    return tT.astype(F), tRT.astype(F)


class Ref:
    """The float64 reference of one (level, pose, affine, cutoff) evaluation.  See the module docstring for what every field holds."""

    def __init__(self, otr, frame, lvl, T7, a, b, cutoff, huber=6.0, ref_a=0.0, ref_b=0.0, gs=True):
        T7 = np.asarray(T7, np.float64)
        self.rs_oracle = rs = otr.calcRes(frame, lvl, T7, a, b, cutoff)
        self.nE = nE = int(rs[1]); self.nSat = nSat = int(round(rs[5] * rs[1])) if nE else 0
        self.nW = nW = nE - nSat; self.npad = (nW + 3) & ~3; self.lvl = lvl
        wp = otr.warped()[:, :nW]
        nid, u, v, dx, dy, res, hw, col = (np.asarray(r, F) for r in wp)
        K4 = otr.K(lvl); fx, fy = F(K4[0]), F(K4[1])
        RKi, t, aLL, bLL, b0 = eval_params(T7, otr.Ki(lvl), a, b, ref_a, ref_b)
        self.aLL, self.bLL = aLL, bLL
        S = np.zeros(48); A = np.zeros(48)
        maxE = F(F(F(2) * F(huber)) * F(cutoff)) - F(F(huber) * F(huber))
        e = ((hw * res) * res) * (F(2) - hw)
        S[IDX_E] = math.fsum(np.asarray(e, np.float64).tolist() + [float(maxE) * nSat])
        A[IDX_E] = float(np.abs(e.astype(np.float64)).sum()) + abs(float(maxE)) * nSat
        self.e = e; self.maxEnergy = maxE
        if gs:
            one, zero = F(1), F(0)
            dxf, dyf = dx * fx, dy * fy
            J = [nid * dxf, nid * dyf, zero - nid * (u * dxf + v * dyf), zero - ((u * v) * dxf + dyf * (one + v * v)),
                 (u * v) * dyf + dxf * (one + u * u), u * dyf - v * dxf, np.full(nW, aLL, F) * (b0 - col), np.full(nW, F(-1)), res]
            J = [np.asarray(j, F) for j in J]
            for k, (r, c) in enumerate(RC):
                term = (J[r] * hw) * J[c]
                S[k] = _fsum(term); A[k] = float(np.abs(term.astype(np.float64)).sum())
        self.n_flow = 0
        if lvl == 0:
            cloud = otr.cloud(0)
            tT, tRT = flow_terms(cloud, K4, otr.Ki(0), RKi, t)
            self.n_flow = len(tT)
            S[IDX_FT], S[IDX_FRT] = _fsum(tT), _fsum(tRT)
            A[IDX_FT], A[IDX_FRT] = float(np.abs(tT.astype(np.float64)).sum()), float(np.abs(tRT.astype(np.float64)).sum())
        self.S, self.A = S, A
        # finalize_res
        fN = float(F(self.n_flow))
        with np.errstate(all="ignore"):
            self.rs = np.array([float(F(S[IDX_E])), float(F(nE)), float(F(S[IDX_FT])) / (fN + 0.1), 0.0,
                                float(F(S[IDX_FRT])) / (fN + 0.1), float(F(nSat) / F(nE)) if nE else float("nan")])
            # finalize_gs
            invn = float(F(1) / F(self.npad)) if self.npad else float("inf")
            self.scale = np.zeros(45)
            H = np.zeros((8, 8)); bb = np.zeros(8)
            for k, (r, c) in enumerate(RC):
                hv = float(F(S[k]))
                if c < 8:
                    H[r, c] = H[c, r] = hv * invn * SC[c] * SC[r]; self.scale[k] = invn * SC[c] * SC[r]
                elif r < 8:
                    bb[r] = hv * invn * SC[r]; self.scale[k] = invn * SC[r]
            self.H, self.b = H, bb
            self.lastRes = math.sqrt(S[IDX_E] / nE) if nE else float("nan")

    # ---------------------------------------------------------------- bounds
    def sum_bound(self, k, m):
        """Bound on |kernel total - S| after the float32 cast, in the units of S (entry k; m points per thread)."""
        mm = 2 * m if k in (IDX_FT, IDX_FRT) else m
        return 1.001 * (mm + 1) * U * self.A[k] + 1e-12 * self.A[k] + 2 * U * abs(self.S[k])

    def check_res(self, rs, m, rep, tag, m_flow=None):
        """rs (calcRes Vec6) against the reference: nE, nSat exact; E and the flow indicators within the bound."""
        assert int(rs[1]) == self.nE, (tag, rs[1], self.nE)
        if self.nE:
            assert int(round(rs[5] * rs[1])) == self.nSat, (tag, rs[5], self.nSat)
        rep.check(tag + " E", abs(rs[0] - self.rs[0]), self.sum_bound(IDX_E, m))
        mf = m if m_flow is None else m_flow
        fN = float(F(self.n_flow)) + 0.1
        rep.check(tag + " flowT", abs(rs[2] - self.rs[2]), self.sum_bound(IDX_FT, mf) / fN)
        rep.check(tag + " flowRT", abs(rs[4] - self.rs[4]), self.sum_bound(IDX_FRT, mf) / fN)

    def check_gs(self, H, b, m, rep, tag):
        """H (8x8), b (8) of calcGSSSE against the reference, entry by entry within the bound."""
        if self.nW == 0:
            assert np.all(np.isnan(H)) and np.all(np.isnan(b)), tag
            return
        for k, (r, c) in enumerate(RC):
            if r == 8:
                continue
            got = H[r, c] if c < 8 else b[r]
            want = self.H[r, c] if c < 8 else self.b[r]
            rep.check(tag + (" H" if c < 8 else " b"), abs(got - want), self.sum_bound(k, m) * abs(self.scale[k]) * (1 + 1e-12) + 1e-300)

    def lastres_bound(self, m):
        if not self.nE or self.S[IDX_E] == 0:
            return 4 * U * abs(self.lastRes) + 1e-30
        return self.lastRes * (self.sum_bound(IDX_E, m) / (2 * self.S[IDX_E]) + 2 * U) * 1.001


class Report:
    """Worst observed error as a fraction of its bound, per check name; every check asserts error <= bound."""

    def __init__(self, title):
        self.title, self.worst = title, {}

    def check(self, name, err, bound):
        assert err <= bound, f"{self.title}: {name}: error {err:.3e} exceeds bound {bound:.3e}"
        r = err / bound if bound > 0 else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), r)

    def print(self):
        items = ", ".join(f"{k} {v:.3f}" for k, v in sorted(self.worst.items()))
        print(f"\n[{self.title}] worst error / bound: {items}")
