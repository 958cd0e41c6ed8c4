// gms_alpha.cuh -- alpha shape and normal estimation of a point cloud (the reference's scripts/create_dummy_mesh.py: open3d's
// CreateFromPointCloudAlphaShape and EstimateNormals), float64 geometry, sm_90a.  include/gms_b200.h states the contract.
//
// Alpha shape without a global triangulation.  Take a triangle f = (a,b,c) with circumcentre c_f, circumradius r_f and unit
// normal n.  Every sphere through a, b, c has its centre at c_f + t n, and a point p lies on the one with
//   t_p = (|p - c_f|^2 - r_f^2) / (2 n.(p - c_f)).
// With T+ = min t_p over points on the + side, T- = max t_p over the - side and beta = sqrt(alpha^2 - r_f^2):
//   f is a Delaunay face iff T- < T+ (and no point in f's plane lies strictly inside its circumcircle);
//   its + tetrahedron (circumradius sqrt(r_f^2 + T+^2)) has circumradius <= alpha iff |T+| <= beta, likewise for -.
// f is output iff it is Delaunay and exactly one side is kept.  Every point that can change that answer lies within 2 alpha of
// c_f: a point with |t_p| <= beta lies on a sphere of radius <= alpha centred within beta of c_f; a + point with t_p < 0 lies
// inside the circumcircle's ball (|p - c_f| < r_f); so a point farther than 2 alpha from c_f has t_p > beta on the + side and
// t_p < -beta on the - side, and can neither change which side is kept nor, when exactly one side is kept, Delaunay-ness.
// With r_f <= alpha every such point lies within 3 alpha of a, and b, c lie within 2 alpha of a.  So the kernels below:
//   1. grid: the cloud's bounds and mean (deterministic two-pass reduction), cells of h = max(3 alpha (1 + 1e-6),
//      extent / (2^21 - 1)), a 63-bit cell key per point, a radix sort of (key, index);
//   2. exact duplicates: a point with an equal point of lower index in its cell takes no further part;
//   3. neighbour lists (CSR, original index order): every live point within 3 alpha ("all"), and the subset of higher index
//      within 2 alpha ("up", segment-sorted by index); count, scan, one host synchronisation to size them, gather;
//   4. faces: one warp per point a; lanes take the pairs (b, c) of its up list in lexicographic order, drop r_f > alpha at once
//      and scan a's all list (staged in shared memory, or read from global memory when longer than GMS_ALPHA_LIST_CAP) for
//      T+ / T-, stopping once T- >= T+.  A count pass marks the referenced points; after the scans and the second host
//      synchronisation an emit pass writes faces in lexicographic order through a ballot, without atomics;
//   5. vertices: the referenced points in ascending index (the count pass's flags, scanned).
// Normals: the same grid at h = radius, the max_nn nearest points by (squared distance, index) within radius in registers and
// local memory, float64 covariance and a cyclic Jacobi eigen-solver.
//
// The predicates below are host + device: tests/hostshim builds them for the CPU.
#pragma once
#include "gms_common.cuh"
#include "../../include/gms_b200.h"     // GMS_ALPHA_LIST_CAP, GMS_NORMALS_MAX_NN

#define GMS_GRID_BITS 21
#define GMS_GRID_MAXC ((1 << GMS_GRID_BITS) - 1)

// ---- shared float64 face predicates
struct GmsAlphaFace {
    double wx, wy, wz;      // w = (b - a) x (c - a), the unnormalised normal
    double cx, cy, cz;      // circumcentre minus a
    double beta2;           // (alpha^2 - r_f^2) / |w|^2: a side is kept iff tau^2 <= beta2, tau = t / |w|
};

// false when (a, b, c) is collinear or r_f > alpha (never output).  u = b - a, v = c - a.
GMS_HD bool gms_alpha_face_setup(double ux, double uy, double uz, double vx, double vy, double vz, double alpha2, GmsAlphaFace& f) {
    const double wx = uy * vz - uz * vy, wy = uz * vx - ux * vz, wz = ux * vy - uy * vx;
    const double w2 = wx * wx + wy * wy + wz * wz;
    if (!(w2 > 0.0)) return false;
    const double u2 = ux * ux + uy * uy + uz * uz, v2 = vx * vx + vy * vy + vz * vz;
    // c = (|u|^2 (v x w) + |v|^2 (w x u)) / (2 |w|^2)
    const double s = 0.5 / w2;
    const double cx = (u2 * (vy * wz - vz * wy) + v2 * (wy * uz - wz * uy)) * s;
    const double cy = (u2 * (vz * wx - vx * wz) + v2 * (wz * ux - wx * uz)) * s;
    const double cz = (u2 * (vx * wy - vy * wx) + v2 * (wx * uy - wy * ux)) * s;
    const double r2 = cx * cx + cy * cy + cz * cz;
    if (r2 > alpha2) return false;
    f.wx = wx; f.wy = wy; f.wz = wz; f.cx = cx; f.cy = cy; f.cz = cz;
    f.beta2 = (alpha2 - r2) / w2;
    return true;
}

// One other point q (minus a): tp = min tau over w.q > 0, tm = max tau over w.q < 0, tau = (|q|^2 - 2 q.c) / (2 w.q);
// a point in the plane (w.q == 0) strictly inside the circumcircle blocks the face.  Returns true once the face is decided
// not Delaunay (blocked or tm >= tp), so the caller can stop.
GMS_HD bool gms_alpha_face_point(const GmsAlphaFace& f, double qx, double qy, double qz, double& tp, double& tm, bool& blocked) {
    const double s = f.wx * qx + f.wy * qy + f.wz * qz;
    const double pw = (qx * qx + qy * qy + qz * qz) - 2.0 * (qx * f.cx + qy * f.cy + qz * f.cz);
    if (s > 0.0) {
        const double t = pw / (2.0 * s);
        tp = t < tp ? t : tp;
    } else if (s < 0.0) {
        const double t = pw / (2.0 * s);
        tm = t > tm ? t : tm;
    } else if (pw < 0.0) {
        blocked = true;
    }
    return blocked || !(tm < tp);
}

// Tie rule: Delaunay needs T- < T+ strictly; a side is kept when tau^2 <= beta2 (circumradius <= alpha); a missing side
// (tau infinite) is never kept.
GMS_HD bool gms_alpha_face_decide(const GmsAlphaFace& f, double tp, double tm, bool blocked) {
    if (blocked || !(tm < tp)) return false;
    const bool kp = tp * tp <= f.beta2, km = tm * tm <= f.beta2;
    return kp != km;
}

// ---- 3x3 symmetric eigen-solver (cyclic Jacobi, float64): the unit eigenvector of the smallest eigenvalue
GMS_HD void gms_sym3_min_eigvec(const double* A6 /* xx xy xz yy yz zz */, double* n) {
    double a[3][3] = {{A6[0], A6[1], A6[2]}, {A6[1], A6[3], A6[4]}, {A6[2], A6[4], A6[5]}};
    double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 32; sweep++) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        const double dia = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
        if (!(off > 1e-36 * dia)) break;
        for (int p = 0; p < 2; p++)
            for (int q = p + 1; q < 3; q++) {
                const double apq = a[p][q];
                if (apq == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; k++) {       // A <- A J (columns p, q)
                    const double akp = a[k][p], akq = a[k][q];
                    a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; k++) {       // A <- J^T A (rows p, q)
                    const double apk = a[p][k], aqk = a[q][k];
                    a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; k++) {       // V <- V J
                    const double vkp = v[k][p], vkq = v[k][q];
                    v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq;
                }
            }
    }
    int m = 0;
    if (a[1][1] < a[m][m]) m = 1;
    if (a[2][2] < a[m][m]) m = 2;
    const double l = sqrt(v[0][m] * v[0][m] + v[1][m] * v[1][m] + v[2][m] * v[2][m]);
    n[0] = v[0][m] / l; n[1] = v[1][m] / l; n[2] = v[2][m] / l;
}

// Sign rule: n.(x - mean(cloud)) >= 0; when that is exactly 0, the largest-magnitude component (the first of equals) is positive.
GMS_HD void gms_normal_orient(double* n, double dx, double dy, double dz) {
    const double d = n[0] * dx + n[1] * dy + n[2] * dz;
    bool flip = d < 0.0;
    if (d == 0.0) {
        int m = 0;
        if (fabs(n[1]) > fabs(n[m])) m = 1;
        if (fabs(n[2]) > fabs(n[m])) m = 2;
        flip = n[m] < 0.0;
    }
    if (flip) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
}

#if defined(__CUDACC__)

#define GMS_GRID_STAT_BLOCKS 256

struct GmsGridStats { double lo[3], hi[3], sum[3]; };
struct GmsGrid { double lo[3], inv_h, mean[3]; };

__device__ __forceinline__ void grid_stats_add(GmsGridStats& s, const GmsGridStats& o) {
    for (int k = 0; k < 3; k++) { s.lo[k] = fmin(s.lo[k], o.lo[k]); s.hi[k] = fmax(s.hi[k], o.hi[k]); s.sum[k] += o.sum[k]; }
}

// the CTA's (256 threads) stats in a fixed order: the same points give the same bits whatever the device's state
__device__ __forceinline__ GmsGridStats grid_stats_cta(GmsGridStats s) {
    __shared__ GmsGridStats part[256];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) grid_stats_add(part[threadIdx.x], part[threadIdx.x + o]);
        __syncthreads();
    }
    return part[0];
}

__global__ void __launch_bounds__(256) k_grid_stats(int P, const float* __restrict__ pts, GmsGridStats* __restrict__ part) {
    GmsGridStats s;
    for (int k = 0; k < 3; k++) { s.lo[k] = INFINITY; s.hi[k] = -INFINITY; s.sum[k] = 0.0; }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x)
        for (int k = 0; k < 3; k++) {
            const double x = pts[3 * (size_t)i + k];
            s.lo[k] = fmin(s.lo[k], x); s.hi[k] = fmax(s.hi[k], x); s.sum[k] += x;
        }
    s = grid_stats_cta(s);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// cell size h = max(hmin, extent / (2^21 - 1)): every coordinate's cell fits 21 bits; cells only grow, so the +-1 cell
// neighbourhood still covers every point within hmin.
__global__ void __launch_bounds__(256) k_grid_fold(int P, const GmsGridStats* __restrict__ part, double hmin, GmsGrid* __restrict__ g) {
    const GmsGridStats s = grid_stats_cta(part[threadIdx.x]);
    if (threadIdx.x == 0) {
        double ext = 0.0;
        for (int k = 0; k < 3; k++) ext = fmax(ext, s.hi[k] - s.lo[k]);
        const double h = fmax(hmin, ext / (double)GMS_GRID_MAXC * (1.0 + 1e-9));
        GmsGrid r;
        for (int k = 0; k < 3; k++) { r.lo[k] = s.lo[k]; r.mean[k] = s.sum[k] / (double)P; }
        r.inv_h = 1.0 / h;
        *g = r;
    }
}

__device__ __forceinline__ int grid_coord(double x, double lo, double inv_h) {
    const double c = floor((x - lo) * inv_h);
    return (int)fmin(fmax(c, 0.0), (double)GMS_GRID_MAXC);
}

__device__ __forceinline__ uint64_t grid_key(int cx, int cy, int cz) {
    return (uint64_t)cz << (2 * GMS_GRID_BITS) | (uint64_t)cy << GMS_GRID_BITS | (uint64_t)cx;
}

__global__ void __launch_bounds__(256) k_grid_keys(int P, const float* __restrict__ pts, const GmsGrid* __restrict__ grid,
                                                   uint64_t* __restrict__ key, uint32_t* __restrict__ idx, float4* __restrict__ p4) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const GmsGrid g = *grid;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    key[i] = grid_key(grid_coord(x, g.lo[0], g.inv_h), grid_coord(y, g.lo[1], g.inv_h), grid_coord(z, g.lo[2], g.inv_h));
    idx[i] = (uint32_t)i;
    p4[i] = make_float4(x, y, z, __int_as_float(i));
}

__global__ void __launch_bounds__(256) k_grid_gather(int P, const float4* __restrict__ p4, const uint32_t* __restrict__ idx_s,
                                                     float4* __restrict__ sorted) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < P) sorted[k] = p4[idx_s[k]];
}

// first position in keys[0, n) with key >= v (upper = false) or key > v (upper = true)
__device__ __forceinline__ int grid_bound(const uint64_t* __restrict__ keys, int n, uint64_t v, bool upper) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const uint64_t k = keys[mid];
        if (upper ? k <= v : k < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Calls f(sorted position) for every point in the 27 cells around `key`: nine runs of three consecutive x cells, each one
// contiguous range of the sorted keys.
template <class F>
__device__ __forceinline__ void grid_visit(const uint64_t* __restrict__ keys_s, int P, uint64_t key, F&& f) {
    const int cx = (int)(key & GMS_GRID_MAXC), cy = (int)(key >> GMS_GRID_BITS & GMS_GRID_MAXC), cz = (int)(key >> (2 * GMS_GRID_BITS));
    for (int z = max(cz - 1, 0); z <= min(cz + 1, GMS_GRID_MAXC); z++)
        for (int y = max(cy - 1, 0); y <= min(cy + 1, GMS_GRID_MAXC); y++) {
            const int b = grid_bound(keys_s, P, grid_key(max(cx - 1, 0), y, z), false);
            const int e = grid_bound(keys_s, P, grid_key(min(cx + 1, GMS_GRID_MAXC), y, z), true);
            for (int k = b; k < e; k++) f(k);
        }
}

__device__ __forceinline__ double alpha_d2(const float4& p, const float4& q) {
    const double dx = (double)q.x - p.x, dy = (double)q.y - p.y, dz = (double)q.z - p.z;
    return dx * dx + dy * dy + dz * dz;
}

// alive[i] = 0 when an equal point of lower index exists (equal points share a cell)
__global__ void __launch_bounds__(256) k_alpha_dedup(int P, const uint64_t* __restrict__ keys_s, const float4* __restrict__ sorted,
                                                     int32_t* __restrict__ alive) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const float4 p = sorted[k];
    const int i = __float_as_int(p.w);
    const uint64_t key = keys_s[k];
    int dup = 0;
    for (int j = grid_bound(keys_s, P, key, false); j < P && keys_s[j] == key; j++) {
        const float4 q = sorted[j];
        if (q.x == p.x && q.y == p.y && q.z == p.z && __float_as_int(q.w) < i) { dup = 1; break; }
    }
    alive[i] = !dup;
}

// Neighbour lists of every live point (thread per sorted position; lists by original index).  COUNT: n_all / n_up;
// otherwise the entries at off_all / off_up.  r_all2 = (3 alpha)^2, r_up2 = (2 alpha)^2, both widened by 1e-9.
template <bool COUNT>
__global__ void __launch_bounds__(256) k_alpha_lists(int P, const uint64_t* __restrict__ keys_s, const float4* __restrict__ sorted,
                                                     const int32_t* __restrict__ alive, double r_all2, double r_up2,
                                                     int64_t* __restrict__ n_all, int64_t* __restrict__ n_up,
                                                     const int64_t* __restrict__ off_all, const int64_t* __restrict__ off_up,
                                                     int32_t* __restrict__ all, int32_t* __restrict__ up) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const float4 p = sorted[k];
    const int i = __float_as_int(p.w);
    if (!alive[i]) {
        if (COUNT) { n_all[i] = 0; n_up[i] = 0; }
        return;
    }
    int64_t ca = COUNT ? 0 : off_all[i], cu = COUNT ? 0 : off_up[i];
    grid_visit(keys_s, P, keys_s[k], [&](int s) {
        const float4 q = sorted[s];
        const int j = __float_as_int(q.w);
        if (j == i || !alive[j]) return;
        const double d2 = alpha_d2(p, q);
        if (!(d2 <= r_all2)) return;
        if (!COUNT) all[ca] = j;
        ca++;
        if (j > i && d2 <= r_up2) {
            if (!COUNT) up[cu] = j;
            cu++;
        }
    });
    if (COUNT) { n_all[i] = ca; n_up[i] = cu; }
}

#define GMS_ALPHA_WARPS 4       // warps per CTA of the face kernel

// One warp per point a.  COUNT: fcount[a] = faces with lowest vertex a, ref[] = 1 for their vertices.  Otherwise: the faces,
// remapped through voff, written from foff[a] on in lexicographic order.
template <bool COUNT>
__global__ void __launch_bounds__(GMS_ALPHA_WARPS * 32) k_alpha_faces(int P, const float4* __restrict__ p4, const int64_t* __restrict__ off_all,
                                                                      const int32_t* __restrict__ all, const int64_t* __restrict__ off_up,
                                                                      const int32_t* __restrict__ up, double alpha2, int64_t* __restrict__ fcount,
                                                                      int32_t* __restrict__ ref, const int64_t* __restrict__ foff,
                                                                      const int32_t* __restrict__ voff, int64_t* __restrict__ faces) {
    __shared__ float4 stage[GMS_ALPHA_WARPS][GMS_ALPHA_LIST_CAP];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int a = blockIdx.x * GMS_ALPHA_WARPS + w;
    if (a >= P) return;
    const int64_t u0 = off_up[a];
    const int m = (int)(off_up[a + 1] - u0);
    int64_t cnt = 0, pos = COUNT ? 0 : foff[a];
    if (m >= 2) {
        const int64_t l0 = off_all[a];
        const int n = (int)(off_all[a + 1] - l0);
        const bool staged = n <= GMS_ALPHA_LIST_CAP;
        if (staged)
            for (int k = lane; k < n; k += 32) stage[w][k] = p4[all[l0 + k]];
        __syncwarp();
        const float4 A = p4[a];
        const double ax = A.x, ay = A.y, az = A.z;
        int i = 0, j = 1 + lane;                        // this lane's pair: index lane of the lexicographic (i, j), i < j
        while (i < m - 1 && j >= m) { i++; j = j - m + i + 1; }
        while (__any_sync(0xffffffffu, i < m - 1)) {
            bool out = false;
            int ib = 0, ic = 0;
            if (i < m - 1) {
                ib = up[u0 + i]; ic = up[u0 + j];
                const float4 B = p4[ib], Cc = p4[ic];
                GmsAlphaFace f;
                if (gms_alpha_face_setup(B.x - ax, B.y - ay, B.z - az, Cc.x - ax, Cc.y - ay, Cc.z - az, alpha2, f)) {
                    double tp = INFINITY, tm = -INFINITY;
                    bool blocked = false;
                    for (int k = 0; k < n; k++) {
                        const float4 q = staged ? stage[w][k] : p4[all[l0 + k]];
                        const int jj = __float_as_int(q.w);
                        if (jj == ib || jj == ic) continue;
                        if (gms_alpha_face_point(f, q.x - ax, q.y - ay, q.z - az, tp, tm, blocked)) break;
                    }
                    out = gms_alpha_face_decide(f, tp, tm, blocked);
                }
                j += 32;
                while (i < m - 1 && j >= m) { i++; j = j - m + i + 1; }
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, out);
            if (COUNT) {
                if (out) { ref[ib] = 1; ref[ic] = 1; }
            } else if (out) {
                const int64_t o = pos + __popc(bal & ((1u << lane) - 1u));
                faces[3 * o] = voff[a]; faces[3 * o + 1] = voff[ib]; faces[3 * o + 2] = voff[ic];
            }
            cnt += __popc(bal);
            pos += __popc(bal);
        }
    }
    if (COUNT && lane == 0) {
        fcount[a] = cnt;
        if (cnt) ref[a] = 1;
    }
}

__global__ void __launch_bounds__(256) k_alpha_index(int P, const int32_t* __restrict__ ref, const int32_t* __restrict__ voff,
                                                     int64_t* __restrict__ index) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P && ref[i]) index[voff[i]] = i;
}

#pragma nv_diag_suppress 549     // bd / bi are read only below c, which counts the entries written
// Normals: thread per sorted position; the max_nn nearest (d2, index) within radius, point itself included.
__global__ void __launch_bounds__(128) k_normals(int P, const uint64_t* __restrict__ keys_s, const float4* __restrict__ sorted,
                                                 const float4* __restrict__ p4, const GmsGrid* __restrict__ grid, double r2,
                                                 int max_nn, float* __restrict__ normals) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const float4 p = sorted[k];
    const int i = __float_as_int(p.w);
    double bd[GMS_NORMALS_MAX_NN];
    int bi[GMS_NORMALS_MAX_NN];
    int c = 0;
    double wd = INFINITY;       // the last kept (d2, index) once the list is full
    int wi = 0x7fffffff;
    grid_visit(keys_s, P, keys_s[k], [&](int s) {
        const float4 q = sorted[s];
        const double d2 = alpha_d2(p, q);
        if (!(d2 <= r2)) return;
        const int j = __float_as_int(q.w);
        if (!(d2 < wd || (d2 == wd && j < wi))) return;
        int t = c < max_nn ? c++ : c - 1;       // insertion into the ascending (d2, index) list
        while (t > 0 && (d2 < bd[t - 1] || (d2 == bd[t - 1] && j < bi[t - 1]))) { bd[t] = bd[t - 1]; bi[t] = bi[t - 1]; t--; }
        bd[t] = d2; bi[t] = j;
        if (c == max_nn) { wd = bd[c - 1]; wi = bi[c - 1]; }
    });
    double n[3] = {0.0, 0.0, 1.0};
    if (c >= 3) {
        double s1[3] = {0.0, 0.0, 0.0}, s2[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int t = 0; t < c; t++) {
            const float4 q = p4[bi[t]];
            const double dx = (double)q.x - p.x, dy = (double)q.y - p.y, dz = (double)q.z - p.z;
            s1[0] += dx; s1[1] += dy; s1[2] += dz;
            s2[0] += dx * dx; s2[1] += dx * dy; s2[2] += dx * dz; s2[3] += dy * dy; s2[4] += dy * dz; s2[5] += dz * dz;
        }
        const double inv = 1.0 / c, mx = s1[0] * inv, my = s1[1] * inv, mz = s1[2] * inv;
        const double cov[6] = {s2[0] * inv - mx * mx, s2[1] * inv - mx * my, s2[2] * inv - mx * mz,
                               s2[3] * inv - my * my, s2[4] * inv - my * mz, s2[5] * inv - mz * mz};
        gms_sym3_min_eigvec(cov, n);
        const GmsGrid g = *grid;
        gms_normal_orient(n, (double)p.x - g.mean[0], (double)p.y - g.mean[1], (double)p.z - g.mean[2]);
    }
    normals[3 * (size_t)i] = (float)n[0]; normals[3 * (size_t)i + 1] = (float)n[1]; normals[3 * (size_t)i + 2] = (float)n[2];
}
#pragma nv_diag_default 549

#endif  // __CUDACC__
