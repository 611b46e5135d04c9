// Exact geometric predicates of the device Delaunay triangulation (csrc/delaunay.cu), for float32 coordinates.
//
// Each predicate first evaluates its determinant in float64 from coordinate differences and keeps the sign when it
// exceeds a static error bound (Shewchuk's stage-A bounds, taken with a factor of 2 of margin).  Otherwise it
// recomputes the determinant exactly: every float32 is an integer multiple of 2^-149 below 2^128, so scaled by
// 2^149 it is an integer of at most 277 bits, and each determinant is a polynomial in those integers.  The exact
// path evaluates it by cofactor expansion in fixed-width two's complement integers (the ring of integers modulo
// 2^(64 L), wide enough that the true value never wraps), so only the sign is read at the end.  For float32 inputs
// nothing over- or underflows in either path: float64 holds every degree-5 term of float32 values.
//
// Conventions (rows are points):
//   orient3d(a, b, c, d) = det[b - a; c - a; d - a]; > 0 is a positively oriented tetrahedron.
//   insphere(a, b, c, d, e) > 0 when e lies strictly inside the circumsphere of a positively oriented (a, b, c, d).
//   orient2d_k(a, b, c) = det[[u v 1]] in the projection k (0: (x, y), 1: (y, z), 2: (x, z)).
//   incircle_k(a, b, c, d) = det[[u v x^2+y^2+z^2 1]]: for coplanar points, incircle_k * orient2d_k(a, b, c) > 0
//   when d lies strictly inside the circle through a, b, c (the projection k must not flatten a, b, c).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define DT_HD __host__ __device__ __forceinline__
#define DT_EXACT __host__ __device__ __noinline__  // the rare exact path stays out of the filters' registers
#else
#define DT_HD inline
#define DT_EXACT inline
#endif

namespace spg {
namespace dt {

// ------------------------------------------------------------------------------ fixed-width integers mod 2^(64 L)
template <int L>
struct Big {
    uint64_t w[L];
};

DT_HD void mul64(uint64_t a, uint64_t b, uint64_t& lo, uint64_t& hi) {
#if defined(__CUDA_ARCH__)
    lo = a * b;
    hi = __umul64hi(a, b);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
}

DT_HD uint32_t f32_bits(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
#endif
}

template <int L>
DT_HD Big<L> big_neg(Big<L> a) {
    uint64_t c = 1;
    for (int i = 0; i < L; ++i) {
        const uint64_t t = ~a.w[i] + c;
        c = (c && t == 0) ? 1 : 0;
        a.w[i] = t;
    }
    return a;
}

// f * 2^149 as an integer (-0 is 0)
template <int L>
DT_HD Big<L> big_f32(float f) {
    Big<L> r;
    for (int i = 0; i < L; ++i) r.w[i] = 0;
    const uint32_t u = f32_bits(f);
    const uint32_t e = (u >> 23) & 0xff;
    uint64_t m = u & 0x7fffff;
    int shift = 0;
    if (e) {
        m |= 0x800000;
        shift = (int)e - 1;
    }
    const int limb = shift >> 6, off = shift & 63;
    r.w[limb] = m << off;
    if (off > 40) r.w[limb + 1] = m >> (64 - off);
    return (u >> 31) ? big_neg(r) : r;
}

// sign extension to a wider width
template <int W, int L>
DT_HD Big<W> big_ext(const Big<L>& a) {
    Big<W> r;
    const uint64_t fill = (a.w[L - 1] >> 63) ? ~0ull : 0ull;
    for (int i = 0; i < W; ++i) r.w[i] = i < L ? a.w[i] : fill;
    return r;
}

template <int L>
DT_HD Big<L> big_add(const Big<L>& a, const Big<L>& b) {
    Big<L> r;
    uint64_t c = 0;
    for (int i = 0; i < L; ++i) {
        const uint64_t s = a.w[i] + b.w[i];
        const uint64_t t = s + c;
        c = (s < a.w[i]) + (t < s);
        r.w[i] = t;
    }
    return r;
}

template <int L>
DT_HD Big<L> big_sub(const Big<L>& a, const Big<L>& b) {
    return big_add(a, big_neg(b));
}

// a * b modulo 2^(64 W), both operands sign-extended first
template <int W, int A, int B>
DT_HD Big<W> big_mul(const Big<A>& a0, const Big<B>& b0) {
    const Big<W> a = big_ext<W>(a0), b = big_ext<W>(b0);
    Big<W> r;
    for (int i = 0; i < W; ++i) r.w[i] = 0;
    for (int i = 0; i < W; ++i) {
        uint64_t carry = 0;
        for (int j = 0; i + j < W; ++j) {
            uint64_t lo, hi;
            mul64(a.w[i], b.w[j], lo, hi);
            uint64_t t = r.w[i + j] + lo;
            hi += t < lo;
            t += carry;
            hi += t < carry;
            r.w[i + j] = t;
            carry = hi;
        }
    }
    return r;
}

template <int L>
DT_HD int big_sign(const Big<L>& a) {
    if (a.w[L - 1] >> 63) return -1;
    for (int i = 0; i < L; ++i)
        if (a.w[i]) return 1;
    return 0;
}

// widths: coordinates 277 bits; degree 2 (minors, lifts) 556; degree 3: 835; degree 4: 1114; degree 5: 1394
typedef Big<5> B1;
typedef Big<9> B2;
typedef Big<14> B3;
typedef Big<18> B4;
typedef Big<22> B5;

struct P3 {
    float x, y, z;
};

DT_HD float coord(const P3& p, int c) { return c == 0 ? p.x : (c == 1 ? p.y : p.z); }

// u_i v_j - u_j v_i
DT_HD B2 minor2(const B1& ui, const B1& vi, const B1& uj, const B1& vj) {
    return big_sub(big_mul<9>(ui, vj), big_mul<9>(uj, vi));
}

DT_HD B2 lift(const P3& p) {
    const B1 x = big_f32<5>(p.x), y = big_f32<5>(p.y), z = big_f32<5>(p.z);
    return big_add(big_add(big_mul<9>(x, x), big_mul<9>(y, y)), big_mul<9>(z, z));
}

// det[[x y z 1]] of four points, the 3x3 minors shared through m3 (m3[t] for the triple leaving out point t)
DT_HD B3 det4_from_m3(const B3 m3[4]) {
    // expansion along the column of ones: signs -, +, -, + for the rows 0..3
    return big_sub(big_add(big_sub(m3[1], m3[0]), m3[3]), m3[2]);
}

// det[[x y z]] of three points
DT_HD B3 det3_xyz(const B1* x, const B1* y, const B1* z, int i, int j, int k) {
    const B2 mjk = minor2(x[j], y[j], x[k], y[k]);
    const B2 mik = minor2(x[i], y[i], x[k], y[k]);
    const B2 mij = minor2(x[i], y[i], x[j], y[j]);
    return big_add(big_sub(big_mul<14>(z[i], mjk), big_mul<14>(z[j], mik)), big_mul<14>(z[k], mij));
}

// det[[x y z 1]] of p[0..3] exactly (= -orient3d)
DT_EXACT int det4_exact_sign(const P3* p) {
    B1 x[4], y[4], z[4];
    for (int i = 0; i < 4; ++i) {
        x[i] = big_f32<5>(p[i].x);
        y[i] = big_f32<5>(p[i].y);
        z[i] = big_f32<5>(p[i].z);
    }
    B3 m3[4];
    m3[0] = det3_xyz(x, y, z, 1, 2, 3);
    m3[1] = det3_xyz(x, y, z, 0, 2, 3);
    m3[2] = det3_xyz(x, y, z, 0, 1, 3);
    m3[3] = det3_xyz(x, y, z, 0, 1, 2);
    return big_sign(det4_from_m3(m3));
}

// det[[x y z w 1]] of p[0..4] exactly (= -insphere)
DT_EXACT int det5_exact_sign(const P3* p) {
    B1 x[5], y[5], z[5];
    for (int i = 0; i < 5; ++i) {
        x[i] = big_f32<5>(p[i].x);
        y[i] = big_f32<5>(p[i].y);
        z[i] = big_f32<5>(p[i].z);
    }
    // the ten triples' 3x3 minors, indexed by the pair (l, m) of points left out, l < m
    B3 m3[5][5];
    for (int l = 0; l < 5; ++l)
        for (int m = l + 1; m < 5; ++m) {
            int t[3], c = 0;
            for (int i = 0; i < 5; ++i)
                if (i != l && i != m) t[c++] = i;
            m3[l][m] = m3[m][l] = det3_xyz(x, y, z, t[0], t[1], t[2]);
        }
    B5 acc;
    for (int i = 0; i < 22; ++i) acc.w[i] = 0;
    for (int r = 0; r < 5; ++r) {
        // det[[x y z 1]] of the four points other than r; its row s leaves out (r, s)
        B3 q[4];
        int c = 0;
        for (int s = 0; s < 5; ++s)
            if (s != r) q[c++] = m3[r][s];
        const B3 d4 = det4_from_m3(q);
        const B5 term = big_mul<22>(lift(p[r]), d4);
        // expansion along the lift column (column 4 of 5): sign (-1)^(r + 4) for the rows 0..4
        acc = (r & 1) ? big_add(acc, term) : big_sub(acc, term);
    }
    return big_sign(acc);
}

// det[[u v 1]] of three points in the projection k
DT_EXACT int orient2d_exact(const P3& a, const P3& b, const P3& c, int k) {
    const int cu = k == 1 ? 1 : 0, cv = k == 0 ? 1 : 2;
    const P3* p[3] = {&a, &b, &c};
    B1 u[3], v[3];
    for (int i = 0; i < 3; ++i) {
        u[i] = big_f32<5>(coord(*p[i], cu));
        v[i] = big_f32<5>(coord(*p[i], cv));
    }
    const B2 d = big_add(big_sub(minor2(u[1], v[1], u[2], v[2]), minor2(u[0], v[0], u[2], v[2])),
                         minor2(u[0], v[0], u[1], v[1]));
    return big_sign(d);
}

// det[[u v w 1]] of four points in the projection k, w the 3D lift
DT_EXACT int incircle_exact(const P3* p, int k) {
    const int cu = k == 1 ? 1 : 0, cv = k == 0 ? 1 : 2;
    B1 u[4], v[4];
    for (int i = 0; i < 4; ++i) {
        u[i] = big_f32<5>(coord(p[i], cu));
        v[i] = big_f32<5>(coord(p[i], cv));
    }
    B4 acc;
    for (int i = 0; i < 18; ++i) acc.w[i] = 0;
    for (int r = 0; r < 4; ++r) {
        int t[3], c = 0;
        for (int i = 0; i < 4; ++i)
            if (i != r) t[c++] = i;
        const B2 a = big_add(big_sub(minor2(u[t[1]], v[t[1]], u[t[2]], v[t[2]]),
                                     minor2(u[t[0]], v[t[0]], u[t[2]], v[t[2]])),
                             minor2(u[t[0]], v[t[0]], u[t[1]], v[t[1]]));
        const B4 term = big_mul<18>(lift(p[r]), a);
        // expansion along the lift column (column 3 of 4): sign (-1)^(r + 3)
        acc = (r & 1) ? big_sub(acc, term) : big_add(acc, term);
    }
    return big_sign(acc);
}

// ------------------------------------------------------------------------------ filtered predicates
constexpr double kEps = 1.1102230246251565e-16;  // 2^-53
constexpr double kO2dBound = 2.0 * (3.0 + 16.0 * kEps) * kEps;
constexpr double kO3dBound = 2.0 * (7.0 + 56.0 * kEps) * kEps;
constexpr double kIspBound = 2.0 * (16.0 + 224.0 * kEps) * kEps;

DT_HD int sgn(double v) { return (v > 0) - (v < 0); }

DT_HD int orient3d(const P3& a, const P3& b, const P3& c, const P3& d) {
    // det[a - d; b - d; c - d] = det[[x y z 1]] = -orient3d
    const double adx = (double)a.x - d.x, ady = (double)a.y - d.y, adz = (double)a.z - d.z;
    const double bdx = (double)b.x - d.x, bdy = (double)b.y - d.y, bdz = (double)b.z - d.z;
    const double cdx = (double)c.x - d.x, cdy = (double)c.y - d.y, cdz = (double)c.z - d.z;
    const double bdxcdy = bdx * cdy, cdxbdy = cdx * bdy;
    const double cdxady = cdx * ady, adxcdy = adx * cdy;
    const double adxbdy = adx * bdy, bdxady = bdx * ady;
    const double det = adz * (bdxcdy - cdxbdy) + bdz * (cdxady - adxcdy) + cdz * (adxbdy - bdxady);
    const double perm = (fabs(bdxcdy) + fabs(cdxbdy)) * fabs(adz) + (fabs(cdxady) + fabs(adxcdy)) * fabs(bdz) +
                        (fabs(adxbdy) + fabs(bdxady)) * fabs(cdz);
    const double bound = kO3dBound * perm;
    if (det > bound || -det > bound) return -sgn(det);
    const P3 p[4] = {a, b, c, d};
    return -det4_exact_sign(p);
}

DT_HD int insphere(const P3& a, const P3& b, const P3& c, const P3& d, const P3& e) {
    const double aex = (double)a.x - e.x, aey = (double)a.y - e.y, aez = (double)a.z - e.z;
    const double bex = (double)b.x - e.x, bey = (double)b.y - e.y, bez = (double)b.z - e.z;
    const double cex = (double)c.x - e.x, cey = (double)c.y - e.y, cez = (double)c.z - e.z;
    const double dex = (double)d.x - e.x, dey = (double)d.y - e.y, dez = (double)d.z - e.z;
    const double aexbey = aex * bey, bexaey = bex * aey, ab = aexbey - bexaey;
    const double bexcey = bex * cey, cexbey = cex * bey, bc = bexcey - cexbey;
    const double cexdey = cex * dey, dexcey = dex * cey, cd = cexdey - dexcey;
    const double dexaey = dex * aey, aexdey = aex * dey, da = dexaey - aexdey;
    const double aexcey = aex * cey, cexaey = cex * aey, ac = aexcey - cexaey;
    const double bexdey = bex * dey, dexbey = dex * bey, bd = bexdey - dexbey;
    const double abc = aez * bc - bez * ac + cez * ab;
    const double bcd = bez * cd - cez * bd + dez * bc;
    const double cda = cez * da + dez * ac + aez * cd;
    const double dab = dez * ab + aez * bd + bez * da;
    const double alift = aex * aex + aey * aey + aez * aez;
    const double blift = bex * bex + bey * bey + bez * bez;
    const double clift = cex * cex + cey * cey + cez * cez;
    const double dlift = dex * dex + dey * dey + dez * dez;
    const double det = (dlift * abc - clift * dab) + (blift * cda - alift * bcd);
    const double az = fabs(aez), bz = fabs(bez), cz = fabs(cez), dz = fabs(dez);
    const double pab = fabs(aexbey) + fabs(bexaey), pbc = fabs(bexcey) + fabs(cexbey);
    const double pcd = fabs(cexdey) + fabs(dexcey), pda = fabs(dexaey) + fabs(aexdey);
    const double pac = fabs(aexcey) + fabs(cexaey), pbd = fabs(bexdey) + fabs(dexbey);
    const double perm = (pcd * bz + pbd * cz + pbc * dz) * alift + (pda * cz + pac * dz + pcd * az) * blift +
                        (pab * dz + pbd * az + pda * bz) * clift + (pbc * az + pac * bz + pab * cz) * dlift;
    const double bound = kIspBound * perm;
    // det = det[[x y z w 1]] = -insphere
    if (det > bound || -det > bound) return -sgn(det);
    const P3 p[5] = {a, b, c, d, e};
    return -det5_exact_sign(p);
}

DT_HD int orient2d(const P3& a, const P3& b, const P3& c, int k) {
    const int cu = k == 1 ? 1 : 0, cv = k == 0 ? 1 : 2;
    const double acu = (double)coord(a, cu) - coord(c, cu), bcv = (double)coord(b, cv) - coord(c, cv);
    const double acv = (double)coord(a, cv) - coord(c, cv), bcu = (double)coord(b, cu) - coord(c, cu);
    const double l = acu * bcv, r = acv * bcu;
    const double det = l - r;
    const double bound = kO2dBound * (fabs(l) + fabs(r));
    if (det > bound || -det > bound) return sgn(det);
    return orient2d_exact(a, b, c, k);
}

// CGAL's coplanar orientation: the first nonzero of the (x, y), (y, z), (x, z) projections' orientations
DT_HD int coplanar_orient(const P3& a, const P3& b, const P3& c) {
    for (int k = 0; k < 3; ++k) {
        const int o = orient2d(a, b, c, k);
        if (o) return o;
    }
    return 0;
}

// ------------------------------------------------------------------------------ symbolic perturbation
// A point is (coordinates, rank), the rank its position in the lexicographic (x, y, z) order of the unique points.

// +1 when e lies inside the perturbed circumsphere of the positively oriented (a, b, c, d), else -1; never 0.
// Exactly on the sphere, the two largest-ranked of the five points are taken from the largest down: if it is e,
// e is outside; else the answer is orient3d with e in that point's place, when it is nonzero.
DT_HD int insphere_perturbed(const P3* v, const int* rank, const P3& e, int re) {
    const int s = insphere(v[0], v[1], v[2], v[3], e);
    if (s) return s;
    int order[5] = {0, 1, 2, 3, 4};
    int rk[5] = {rank[0], rank[1], rank[2], rank[3], re};
    for (int i = 1; i < 5; ++i)  // ascending by rank
        for (int j = i; j > 0 && rk[order[j]] < rk[order[j - 1]]; --j) {
            const int t = order[j];
            order[j] = order[j - 1];
            order[j - 1] = t;
        }
    for (int i = 4; i > 2; --i) {
        const int w = order[i];
        if (w == 4) return -1;
        P3 q[4] = {v[0], v[1], v[2], v[3]};
        q[w] = e;
        const int o = orient3d(q[0], q[1], q[2], q[3]);
        if (o) return o;
    }
    return -1;  // unreachable for a non-flat (a, b, c, d)
}

// +1 when d, coplanar with the triangle (a, b, c), lies inside its perturbed circumcircle, else -1.  The same
// scheme in the plane: the three largest-ranked of the four points from the largest down; d itself means outside,
// else the coplanar orientation with d in that point's place, times the triangle's.
DT_HD int incircle_perturbed(const P3* v, const int* rank, const P3& d, int rd) {
    int k = 0, local = 0;
    for (; k < 3; ++k) {
        local = orient2d(v[0], v[1], v[2], k);
        if (local) break;
    }
    const P3 p[4] = {v[0], v[1], v[2], d};
    const int ic = incircle_exact(p, k);
    if (ic) return ic * local;
    int order[4] = {0, 1, 2, 3};
    int rk[4] = {rank[0], rank[1], rank[2], rd};
    for (int i = 1; i < 4; ++i)
        for (int j = i; j > 0 && rk[order[j]] < rk[order[j - 1]]; --j) {
            const int t = order[j];
            order[j] = order[j - 1];
            order[j - 1] = t;
        }
    for (int i = 3; i > 0; --i) {
        const int w = order[i];
        if (w == 3) return -1;
        P3 q[3] = {v[0], v[1], v[2]};
        q[w] = d;
        const int o = coplanar_orient(q[0], q[1], q[2]);
        if (o) return o * local;
    }
    return -1;
}

}  // namespace dt
}  // namespace spg
