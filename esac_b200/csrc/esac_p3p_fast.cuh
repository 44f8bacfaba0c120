// Branch-free float P3P used ONLY as the rejection prefilter of the sampling stage (hyp.cu).
//
// Same mathematics as p3p_lambdas<> in esac_geom.cuh (pencil of the two distance conics, one degenerate member,
// two lines, line-conic intersections), specialised for throughput: one real root of the cubic (any real root is
// enough whenever the P3P has a real solution), no loops over dynamically sized sets, no dynamically indexed arrays
// (3-way selects instead), reciprocal / rsqrt approximations, and NO data-dependent branch: every "this try certainly
// fails" / "this try goes to the exact path" exit of the straightforward formulation is a mask that latches the
// verdict, and the arithmetic simply runs on (garbage after a decision is harmless), so a warp never diverges on it.
// The code is written over a value pack (Pack1: one try per thread; a pack of two tries side by side in a float2 paid
// on Blackwell's packed fp32x2 pipe and was measured slower on the H100, which has none).  Every decision that is
// numerically borderline returns "may pass", i.e. hands the try to the exact fp64 path; the invariant "an accepted try
// is never rejected here" is what tests/test_host_geom.py::test_float_prefilter_never_rejects_an_accepted_try checks on
// random draws, and tests/test_host_minimal_sets.py (host compile) and tests/test_gpu_minimal_sets.py (device compile)
// on crafted ill-conditioned sets.
#pragma once
#include "esac_geom.cuh"

namespace esacb200 {

// ---- value packs: W tries side by side ---------------------------------------------------------------------------------
struct Pack1 {
    float a;
    static constexpr int W = 1;
};
struct Mask1 {
    bool a;
};
template <typename P> struct MaskOf;
template <> struct MaskOf<Pack1> { typedef Mask1 type; };

ESAC_HD Pack1 bc1(float x) { Pack1 r; r.a = x; return r; }
template <typename P> ESAC_HD P bc(float x);
template <> ESAC_HD Pack1 bc<Pack1>(float x) { return bc1(x); }

// arithmetic
ESAC_HD Pack1 operator+(Pack1 x, Pack1 y) { return bc1(x.a + y.a); }
ESAC_HD Pack1 operator-(Pack1 x, Pack1 y) { return bc1(x.a - y.a); }
ESAC_HD Pack1 operator*(Pack1 x, Pack1 y) { return bc1(x.a * y.a); }
ESAC_HD Pack1 operator-(Pack1 x) { return bc1(-x.a); }
ESAC_HD Pack1 fma_(Pack1 x, Pack1 y, Pack1 z) { return bc1(fmaf(x.a, y.a, z.a)); }

// per-lane scalar functions
#define ESAC_PACK_UNARY(name, expr) \
    ESAC_HD Pack1 name(Pack1 p) { float x = p.a; return bc1(expr); }
ESAC_PACK_UNARY(abs_, fabsf(x))
ESAC_PACK_UNARY(rcp_, Num<float>::div_(1.f, x))
ESAC_PACK_UNARY(sqrt_, Num<float>::sqrt_(x))
ESAC_PACK_UNARY(rsqrt_, rsqrtf(x))
ESAC_PACK_UNARY(cbrt_, cbrtf(x))
#undef ESAC_PACK_UNARY
ESAC_HD Pack1 max_(Pack1 x, Pack1 y) { return bc1(fmaxf(x.a, y.a)); }
ESAC_HD Pack1 min_(Pack1 x, Pack1 y) { return bc1(fminf(x.a, y.a)); }

// comparisons and masks
#define ESAC_PACK_CMP(name, op) \
    ESAC_HD Mask1 name(Pack1 x, Pack1 y) { Mask1 m; m.a = x.a op y.a; return m; }
ESAC_PACK_CMP(lt_, <)
ESAC_PACK_CMP(le_, <=)
ESAC_PACK_CMP(gt_, >)
ESAC_PACK_CMP(ge_, >=)
#undef ESAC_PACK_CMP
ESAC_HD Mask1 operator&(Mask1 x, Mask1 y) { Mask1 m; m.a = x.a && y.a; return m; }
ESAC_HD Mask1 operator|(Mask1 x, Mask1 y) { Mask1 m; m.a = x.a || y.a; return m; }
ESAC_HD Mask1 operator!(Mask1 x) { Mask1 m; m.a = !x.a; return m; }
ESAC_HD Mask1 mask1(bool v) { Mask1 m; m.a = v; return m; }
template <typename M> ESAC_HD M splat(bool v);
template <> ESAC_HD Mask1 splat<Mask1>(bool v) { return mask1(v); }
ESAC_HD bool all_(Mask1 m) { return m.a; }
ESAC_HD Pack1 sel(Mask1 m, Pack1 x, Pack1 y) { return bc1(m.a ? x.a : y.a); }
ESAC_HD Mask1 nan_(Pack1 x) { return mask1(!(x.a == x.a)); }

// index of the largest of three magnitudes (ties: the first), as two masks: is0, is1 (else 2)
template <typename P, typename M>
ESAC_HD void argmax3(P a0, P a1, P a2, M& is0, M& is1) {
    is0 = ge_(a0, a1) & ge_(a0, a2);
    is1 = !is0 & ge_(a1, a2);
}
template <typename P, typename M>
ESAC_HD P sel3(M is0, M is1, P v0, P v1, P v2) { return sel(is0, v0, sel(is1, v1, v2)); }

// Intersections of the line {lam : l.lam = 0} with the conic lam^T D lam = 0 (D symmetric: d00 d01 d02 d11 d12 d22).
// Writes two direction vectors; ok = a real intersection exists; unc is raised on borderline signs.
template <typename P, typename M>
ESAC_HD void fast_line_conic(P l0, P l1, P l2, P d00, P d01, P d02, P d11, P d12, P d22, P o[2][3], M& ok, M& unc) {
    using N = Num<float>;
    const P zero = bc<P>(0.f), one = bc<P>(1.f), two = bc<P>(2.f);
    const P a0 = abs_(l0), a1 = abs_(l1), a2 = abs_(l2);
    M k0, k1;
    argmax3(a0, a1, a2, k0, k1);
    // permuted coordinates (i, j, k) = (k+1, k+2, k)
    const P li = sel3(k0, k1, l1, l2, l0), lj = sel3(k0, k1, l2, l0, l1), lk = sel3(k0, k1, l0, l1, l2);
    const M lk_ok = gt_(abs_(lk), zero);
    const P Dii = sel3(k0, k1, d11, d22, d00), Djj = sel3(k0, k1, d22, d00, d11), Dkk = sel3(k0, k1, d00, d11, d22);
    const P Dij = sel3(k0, k1, d12, d02, d01), Dik = sel3(k0, k1, d01, d12, d02), Djk = sel3(k0, k1, d02, d01, d12);
    const P ilk = rcp_(lk);
    const P r = li * ilk, s = lj * ilk;
    const P A = Dii - two * r * Dik + r * r * Dkk;
    const P B = Dij - s * Dik - r * Djk + r * s * Dkk;
    const P C = Djj - two * s * Djk + s * s * Dkk;
    P disc = B * B - A * C;
    const P mag = B * B + abs_(A * C);
    // A, B and C themselves come out of cancelling sums (near the danger cylinder C << its terms), and the line carries
    // the error of the cubic's float root: the sign of disc is only known beyond the error those terms propagate into it
    const P sA = abs_(Dii) + two * abs_(r * Dik) + r * r * abs_(Dkk);
    const P sB = abs_(Dij) + abs_(s * Dik) + abs_(r * Djk) + abs_(r * s * Dkk);
    const P sC = abs_(Djj) + two * abs_(s * Djk) + s * s * abs_(Dkk);
    const P derr = two * abs_(B) * sB + abs_(A) * sC + abs_(C) * sA;
    unc = unc | !lk_ok | (lk_ok & lt_(abs_(disc), bc<P>(N::kUncertain) * (mag + derr)));
    const M real = !lt_(disc, -(bc<P>(N::kDiscTol) * mag));
    disc = max_(disc, zero);
    const P sq = sqrt_(disc);
    const P q = -(B + sel(ge_(B, zero), sq, -sq));
    const M useA = ge_(abs_(A), abs_(C));
    const P den = sel(useA, A, C), oth = sel(useA, C, A);
    const M den_ok = gt_(abs_(den), zero);
    unc = unc | (lk_ok & real & !den_ok);
    const P r0 = q * rcp_(den);
    const M q_nz = !(ge_(q, zero) & le_(q, zero));  // q != 0
    const P r1 = sel(q_nz, oth * rcp_(q), r0);
    ok = lk_ok & real & den_ok;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
        const P rt = t == 0 ? r0 : r1;
        const P al = sel(useA, rt, one), be = sel(useA, one, rt);
        const P vi = al, vj = be, vk = -(r * al) - s * be;
        o[t][0] = sel3(k0, k1, vk, vj, vi);
        o[t][1] = sel3(k0, k1, vi, vk, vj);
        o[t][2] = sel3(k0, k1, vj, vi, vk);
    }
}

// 4th-point error band, in units of tau, inside which the exact path decides.  It covers the float error of a
// well-conditioned P3P only: near the danger cylinder a float root can miss the 4th point by many tau (no margin up to
// 16 tau was enough there), so those tries are sent to the exact path by the uncertainty latches above and below instead
// (tests/test_host_minimal_sets.py).  The float error of the 4th point is in absolute pixels, though, not in units of tau:
// on make_scene's maps the host compile's float 4th point missed the exact one by up to 0.76 px among accepted tries (at
// tau = 0.5 a try whose exact 4th point is 0.45 px off needed a band of 1.21 px; at tau = 0.05 on a world-offset map,
// 0.37 px), so below tau ~ 0.6 px a band of 2 tau threw away tries the exact path accepts.  The device compile (MUFU
// approximations, its own FMA contraction) errs differently but as much: on an H100, injected sub-pixel tries (about 40k
// accepted random true-expert draws and 12k accepted crafted sets at tau 0.05 - 1) lost 5 accepted tries with 2 tau
// alone, 1 with a floor of 1 px and none with 2 px.  The band is therefore max(kPrefilterMargin tau, kPrefilterFloorPx):
// the floor is twice the smallest one that held on the device and about five times the largest host discrepancy, and it
// is at or below 2 tau for every tau >= 2 px, so at the default tau = 10 the prefilter's verdicts are unchanged
// (tests/test_host_thresholds.py, tests/test_gpu_thresholds.py).  Below tau = 2 px the exact path judges the tries within
// 4 px, as many as at tau = 2.
constexpr float kPrefilterMargin = 2.f;
constexpr float kPrefilterFloorPx = 4.f;
constexpr float kPrefilterNeedle = 0.02f;  // shortest / longest squared side below which the triangle goes to the exact path

// obj[i][c] / img[i][c]: point i, coordinate c, of the W tries of the pack.  Returns, per try, false only when the try
// certainly fails the 4-point gate.  `hint` is raised, per try, when the try is all but certain to pass: a root that is
// used and trusted (accurate residual, scale ok, no depth near a sign change) brings the 4th point within hint_frac * tau,
// and no latch sent the set to the exact path as ill-conditioned.  hint implies the returned mask; it is never a verdict
// (hint_frac = 0: never raised).
template <typename P>
ESAC_HD typename MaskOf<P>::type p3p_may_pass_pack(const P obj[4][3], const P img[4][2], float f, float ppx, float ppy, float tau,
                                                   float margin, float needle, float hint_frac, typename MaskOf<P>::type& hint) {
    typedef typename MaskOf<P>::type M;
    using N = Num<float>;
    const P zero = bc<P>(0.f), one = bc<P>(1.f), two = bc<P>(2.f);
    M decided = splat<M>(false), verdict = splat<M>(false);
    // latch: lanes where `cond` holds and nothing was decided before get `value`
#define ESAC_LATCH(cond, value)                         \
    {                                                   \
        const M c_ = (cond) & !decided;                 \
        verdict = (verdict & !c_) | (c_ & (value));     \
        decided = decided | c_;                         \
    }
    const M yes = splat<M>(true), no = splat<M>(false);
    // ---- bearings, recentred scene points --------------------------------------------------------------------
    P y[3][3], x1[3], x2[3], x3[3];
    const P ifx = bc<P>(N::div_(1.f, f)), vppx = bc<P>(ppx), vppy = bc<P>(ppy);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const P bx = (img[i][0] - vppx) * ifx, by = (img[i][1] - vppy) * ifx;
        const P n = rsqrt_(fma_(bx, bx, fma_(by, by, one)));
        y[i][0] = bx * n; y[i][1] = by * n; y[i][2] = n;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) { x1[c] = obj[1][c] - obj[0][c]; x2[c] = obj[2][c] - obj[0][c]; x3[c] = obj[3][c] - obj[0][c]; }
    const P a12 = x1[0] * x1[0] + x1[1] * x1[1] + x1[2] * x1[2];
    const P a13 = x2[0] * x2[0] + x2[1] * x2[1] + x2[2] * x2[2];
    const P e0 = x1[0] - x2[0], e1 = x1[1] - x2[1], e2 = x1[2] - x2[2];
    const P a23 = e0 * e0 + e1 * e1 + e2 * e2;
    const P amax = max_(a12, max_(a13, a23)), amin = min_(a12, min_(a13, a23));
    // all-zero: certain reject; NaN / huge: exact path
    ESAC_LATCH(nan_(amax), yes)
    ESAC_LATCH(!gt_(amax, zero), no)
    ESAC_LATCH(!lt_(amax, bc<P>(1e30f)), yes)
    const P c12 = y[0][0] * y[1][0] + y[0][1] * y[1][1] + y[0][2] * y[1][2];
    const P c13 = y[0][0] * y[2][0] + y[0][1] * y[2][1] + y[0][2] * y[2][2];
    const P c23 = y[1][0] * y[2][0] + y[1][1] * y[2][1] + y[1][2] * y[2][2];
    const P cm = max_(abs_(c12), max_(abs_(c13), abs_(c23)));
    ESAC_LATCH(lt_(amin, bc<P>(needle) * amax) | gt_(cm, bc<P>(0.9999f)), yes)  // needle triangle / nearly parallel bearings
    const P iam = rcp_(amax);
    const P s12 = a12 * iam, s13 = a13 * iam, s23 = a23 * iam;
    // ---- the two conics (symmetric storage 00 01 02 11 12 22) ------------------------------------------------
    const P p00 = s23, p01 = -(s23 * c12), p11 = s23 - s12, p12 = s12 * c23, p22 = -s12;                  // D1 (p02 = 0)
    const P q00 = s23, q02 = -(s23 * c13), q11 = -s13, q12 = s13 * c23, q22 = s23 - s13;                  // D2 (q01 = 0)
    // adjugates (symmetric), with the structural zeros p02 = q01 = 0 written out
    const P P00 = p11 * p22 - p12 * p12, P01 = -(p01 * p22), P02 = p01 * p12;
    const P P11 = p00 * p22, P12 = -(p00 * p12), P22 = p00 * p11 - p01 * p01;
    const P Q00 = q11 * q22 - q12 * q12, Q01 = q02 * q12, Q02 = -(q02 * q11);
    const P Q11 = q00 * q22 - q02 * q02, Q12 = -(q00 * q12), Q22 = q00 * q11;
    const P k0 = p00 * P00 + p01 * P01;
    const P k3 = q00 * Q00 + q02 * Q02;
    const P k1 = P00 * q00 + P11 * q11 + P22 * q22 + two * (P02 * q02 + P12 * q12);  // tr(adj(D1) D2)
    const P k2 = Q00 * p00 + Q11 * p11 + Q22 * p22 + two * (Q01 * p01 + Q12 * p12);  // tr(D1 adj(D2))
    const P ksc = abs_(k3) + abs_(k2) + abs_(k1) + abs_(k0);
    ESAC_LATCH(!gt_(abs_(k3), bc<P>(1e-4f) * ksc), yes)  // (nearly) degenerate cubic: exact path
    // ---- one real root of k3 g^3 + k2 g^2 + k1 g + k0 ---------------------------------------------------------
    const P ik3 = rcp_(k3);
    const P a = k2 * ik3, b = k1 * ik3, c = k0 * ik3;
    // Depressed form t^3 - 3 Q t + 2 R = 0 (t = g + a/3).  Newton from outside the root bound |t| <= 2 max(sqrt|Q|, cbrt|R|),
    // on the side of the inflection point where the cubic still has to cross zero: monotone convergence to a real root,
    // with no dependence on the (cancellation-prone) sign of the discriminant and no divergent branches.
    const P three = bc<P>(3.f);
    const P Qq = (a * a - three * b) * bc<P>(1.f / 9.f);
    const P Rr = (two * a * a * a - bc<P>(9.f) * a * b + bc<P>(27.f) * c) * bc<P>(1.f / 54.f);
    const P m3 = max_(sqrt_(abs_(Qq)), cbrt_(abs_(Rr)));
    P t = sel(gt_(Rr, zero), bc<P>(-2.002f), bc<P>(2.002f)) * m3;
#pragma unroll
    for (int it = 0; it < 10; ++it) {
        const P fv = (t * t - three * Qq) * t + two * Rr, dv = three * (t * t - Qq);
        t = t - sel(gt_(abs_(dv), zero), fv * rcp_(dv), zero);
    }
    P g = t - a * bc<P>(1.f / 3.f);
    {   // one polishing step on the original monic cubic
        const P fv = ((g + a) * g + b) * g + c, dv = (three * g + two * a) * g + b;
        g = g - sel(gt_(abs_(dv), zero), fv * rcp_(dv), zero);
    }
    ESAC_LATCH(nan_(g), yes)
    {   // a near-multiple root (two base points of the pencil close together: the danger cylinder) is only known to
        // ~sqrt(eps) in float, and so are the lines built from it: exact path
        const P dv = (three * g + two * a) * g + b, ag = abs_(g);
        ESAC_LATCH(lt_(abs_(dv), bc<P>(1e-3f) * ((three * ag + two * abs_(a)) * ag + abs_(b))), yes)
    }
    // ---- degenerate member D0 and the other conic -------------------------------------------------------------
    const M small = le_(abs_(g), one);
    const P w1 = sel(small, one, rcp_(g)), w2 = sel(small, g, one);
    const P d00 = w1 * p00 + w2 * q00, d01 = w1 * p01, d02 = w2 * q02;
    const P d11 = w1 * p11 + w2 * q11, d12 = w1 * p12 + w2 * q12, d22 = w1 * p22 + w2 * q22;
    const P o00 = sel(small, q00, p00), o01 = sel(small, zero, p01), o02 = sel(small, q02, zero);
    const P o11 = sel(small, q11, p11), o12 = sel(small, q12, p12), o22 = sel(small, q22, p22);
    // adj(D0) = -p p^T for a real line pair
    const P B00 = d11 * d22 - d12 * d12, B01 = d02 * d12 - d01 * d22, B02 = d01 * d12 - d02 * d11;
    const P B11 = d00 * d22 - d02 * d02, B12 = d01 * d02 - d00 * d12, B22 = d00 * d11 - d01 * d01;
    M ib0, ib1;
    argmax3(abs_(B00), abs_(B11), abs_(B22), ib0, ib1);
    const P bii = sel3(ib0, ib1, B00, B11, B22);
    const P nD = abs_(d00) + abs_(d11) + abs_(d22) + two * (abs_(d01) + abs_(d02) + abs_(d12));
    // D0 must be (numerically) singular; it is not when the cubic has a near-multiple root and the float root is off
    ESAC_LATCH(gt_(abs_(d00 * B00 + d01 * B01 + d02 * B02), bc<P>(1e-4f) * nD * nD * nD), yes)
    ESAC_LATCH(lt_(abs_(bii), bc<P>(N::kUncertain) * nD * nD), yes)  // rank deficiency / sign of bii not trustworthy
    ESAC_LATCH(!lt_(bii, zero), no)                                   // complex line pair: no real P3P solution
    const P isq = rsqrt_(-bii);
    const P pv0 = sel3(ib0, ib1, B00, B01, B02) * isq, pv1 = sel3(ib0, ib1, B01, B11, B12) * isq, pv2 = sel3(ib0, ib1, B02, B12, B22) * isq;
    // C = D0 + [p]x = 2 m l^T (rank 1): take the row and the column through its largest entry
    const P Cm[3][3] = {{d00, d01 - pv2, d02 + pv1}, {d01 + pv2, d11, d12 - pv0}, {d02 - pv1, d12 + pv0, d22}};
    P best = bc<P>(-1.f);
    P L0 = zero, L1 = zero, L2 = zero, M0 = zero, M1 = zero, M2 = zero;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
            const P v = abs_(Cm[r][cc]);
            const M up = gt_(v, best);
            best = sel(up, v, best);
            L0 = sel(up, Cm[r][0], L0); L1 = sel(up, Cm[r][1], L1); L2 = sel(up, Cm[r][2], L2);
            M0 = sel(up, Cm[0][cc], M0); M1 = sel(up, Cm[1][cc], M1); M2 = sel(up, Cm[2][cc], M2);
        }
    ESAC_LATCH(!gt_(best, zero), yes)
    // ---- up to four depth directions ---------------------------------------------------------------------------
    P dir[4][3];
    M unc = no, okL, okM;
    fast_line_conic(L0, L1, L2, o00, o01, o02, o11, o12, o22, &dir[0], okL, unc);
    fast_line_conic(M0, M1, M2, o00, o01, o02, o11, o12, o22, &dir[2], okM, unc);
    ESAC_LATCH(unc, yes)
    ESAC_LATCH(!okL & !okM, no)
    // ---- 4th point in the frame of the scene triangle ---------------------------------------------------------
    P nrm[3];
    nrm[0] = x1[1] * x2[2] - x1[2] * x2[1];
    nrm[1] = x1[2] * x2[0] - x1[0] * x2[2];
    nrm[2] = x1[0] * x2[1] - x1[1] * x2[0];
    const P g12 = x1[0] * x2[0] + x1[1] * x2[1] + x1[2] * x2[2];
    const P nn = nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2];
    const P det = a12 * a13 - g12 * g12;
    ESAC_LATCH(!gt_(det, bc<P>(1e-6f) * a12 * a13) | !gt_(nn, zero), yes)
    const P v1 = x3[0] * x1[0] + x3[1] * x1[1] + x3[2] * x1[2], v2 = x3[0] * x2[0] + x3[1] * x2[1] + x3[2] * x2[2];
    const P idet = rcp_(det);
    const P al = (v1 * a13 - v2 * g12) * idet, be = (v2 * a12 - v1 * g12) * idet;
    const P ga = (x3[0] * nrm[0] + x3[1] * nrm[1] + x3[2] * nrm[2]) * rcp_(nn);
    const float lim = fmaxf(margin * tau, kPrefilterFloorPx), hlim = hint_frac * tau;
    const P lim2 = bc<P>(lim * lim), hlim2 = bc<P>(hlim * hlim);
    const P sa = sqrt_(amax);
    const P vf = bc<P>(f);
    M pass = no, near = no;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const M live = s < 2 ? okL : okM;
        P l0 = dir[s][0], l1 = dir[s][1], l2 = dir[s][2];
        const P q12 = l0 * l0 + l1 * l1 - two * c12 * l0 * l1;
        const P q13 = l0 * l0 + l2 * l2 - two * c13 * l0 * l2;
        const P q23 = l1 * l1 + l2 * l2 - two * c23 * l1 * l2;
        const M m12 = ge_(q12, q13) & ge_(q12, q23), m13 = !m12 & ge_(q13, q23);
        const P sc2 = sel3(m12, m13, s12, s13, s23) * rcp_(sel3(m12, m13, q12, q13, q23));
        const M scale_ok = gt_(sc2, zero) & lt_(sc2, bc<P>(1e30f));
        P sc = sqrt_(sc2);
        const P mx = max_(abs_(l0), max_(abs_(l1), abs_(l2)));
        const P ku = bc<P>(N::kUncertain) * mx;
        const M near0 = lt_(abs_(l0), ku) | lt_(abs_(l1), ku) | lt_(abs_(l2), ku);
        const M pos3 = gt_(l0, zero) & gt_(l1, zero) & gt_(l2, zero), neg3 = lt_(l0, zero) & lt_(l1, zero) & lt_(l2, zero);
        sc = sel(neg3, -sc, sc);
        const M signs_ok = pos3 | neg3;
        pass = pass | (live & scale_ok & near0);  // a depth changes sign within the error band: exact path
        const M use = live & scale_ok & signs_ok;
        l0 = l0 * sc; l1 = l1 * sc; l2 = l2 * sc;
        const P res = abs_(l0 * l0 + l1 * l1 - two * c12 * l0 * l1 - s12) + abs_(l0 * l0 + l2 * l2 - two * c13 * l0 * l2 - s13) +
                      abs_(l1 * l1 + l2 * l2 - two * c23 * l1 * l2 - s23);
        const M accurate = lt_(res, bc<P>(1e-4f) * (l0 * l0 + l1 * l1 + l2 * l2 + one));
        pass = pass | (use & !accurate);  // inaccurate candidate: not trusted
        P P0[3], u1[3], u2[3], m[3];
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
            P0[cc] = l0 * sa * y[0][cc];
            u1[cc] = l1 * sa * y[1][cc] - P0[cc];
            u2[cc] = l2 * sa * y[2][cc] - P0[cc];
        }
        m[0] = u1[1] * u2[2] - u1[2] * u2[1];
        m[1] = u1[2] * u2[0] - u1[0] * u2[2];
        m[2] = u1[0] * u2[1] - u1[1] * u2[0];
        const P xc = P0[0] + al * u1[0] + be * u2[0] + ga * m[0];
        const P yc = P0[1] + al * u1[1] + be * u2[1] + ga * m[1];
        const P zc = P0[2] + al * u1[2] + be * u2[2] + ga * m[2];
        const P iz = rcp_(zc);
        const P du = vppx + vf * xc * iz - img[3][0], dv = vppy + vf * yc * iz - img[3][1];
        const P e = du * du + dv * dv;
        pass = pass | (use & !gt_(e, lim2));  // close enough (or NaN/inf): let the exact path decide
        near = near | (use & accurate & !near0 & le_(e, hlim2));
    }
    hint = near & !decided & pass;  // every earlier latch either rejected or forwarded an ill-conditioned set
    ESAC_LATCH(yes, pass)
#undef ESAC_LATCH
    return verdict;
}
template <typename P>
ESAC_HD typename MaskOf<P>::type p3p_may_pass_pack(const P obj[4][3], const P img[4][2], float f, float ppx, float ppy, float tau,
                                                   float margin = kPrefilterMargin, float needle = kPrefilterNeedle) {
    typename MaskOf<P>::type hint;
    return p3p_may_pass_pack<P>(obj, img, f, ppx, ppy, tau, margin, needle, 0.f, hint);
}

// one try (tail_kernel, host test hooks)
ESAC_HD bool p3p_may_pass_fast(const float obj[4][3], const float img[4][2], float f, float ppx, float ppy, float tau,
                               float margin = kPrefilterMargin, float needle = kPrefilterNeedle) {
    Pack1 o[4][3], im[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int c = 0; c < 3; ++c) o[i][c] = bc1(obj[i][c]);
        im[i][0] = bc1(img[i][0]); im[i][1] = bc1(img[i][1]);
    }
    return p3p_may_pass_pack<Pack1>(o, im, f, ppx, ppy, tau, margin, needle).a;
}
// ... and its "near-certain" hint (prefilter_kernel, host test hooks): returns may-pass, `hint` implies it
ESAC_HD bool p3p_may_pass_hint(const float obj[4][3], const float img[4][2], float f, float ppx, float ppy, float tau,
                               float hint_frac, bool& hint, float margin = kPrefilterMargin, float needle = kPrefilterNeedle) {
    Pack1 o[4][3], im[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int c = 0; c < 3; ++c) o[i][c] = bc1(obj[i][c]);
        im[i][0] = bc1(img[i][0]); im[i][1] = bc1(img[i][1]);
    }
    Mask1 h;
    const bool pass = p3p_may_pass_pack<Pack1>(o, im, f, ppx, ppy, tau, margin, needle, hint_frac, h).a;
    hint = h.a;
    return pass;
}

}  // namespace esacb200
