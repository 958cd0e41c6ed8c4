// tests/hostshim/alpha_shim.cpp -- the PRODUCT's float64 alpha-shape face predicates and normal maths (csrc/gms_alpha.cuh)
// built for the CPU, driven by a brute-force neighbour search, so the face classification and the eigen-solver can be checked
// against the Qhull oracle on a machine with no GPU.  TEST-ONLY: the product path is the CUDA kernels.
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "../../gaussian-mesh-splatting_b200/csrc/gms_alpha.cuh"

extern "C" {

// faces (a < b < c, lexicographic) of the points pts[P,3] (float32, no duplicates); returns the count, writes up to cap.
int64_t shim_alpha_faces(int P, const float* pts, double alpha, int64_t* faces, int64_t cap) {
    const double alpha2 = alpha * alpha, r_all2 = 9.0 * alpha2 * (1.0 + 1e-9), r_up2 = 4.0 * alpha2 * (1.0 + 1e-9);
    auto d2 = [&](int i, int j) {
        const double dx = (double)pts[3 * j] - pts[3 * i], dy = (double)pts[3 * j + 1] - pts[3 * i + 1], dz = (double)pts[3 * j + 2] - pts[3 * i + 2];
        return dx * dx + dy * dy + dz * dz;
    };
    int64_t F = 0;
    for (int a = 0; a < P; a++) {
        std::vector<int> all, up;
        for (int j = 0; j < P; j++) {
            if (j == a) continue;
            const double d = d2(a, j);
            if (!(d <= r_all2)) continue;
            all.push_back(j);
            if (j > a && d <= r_up2) up.push_back(j);
        }
        const double ax = pts[3 * a], ay = pts[3 * a + 1], az = pts[3 * a + 2];
        for (size_t i = 0; i < up.size(); i++)
            for (size_t k = i + 1; k < up.size(); k++) {
                const int b = up[i], c = up[k];
                GmsAlphaFace f;
                if (!gms_alpha_face_setup(pts[3 * b] - ax, pts[3 * b + 1] - ay, pts[3 * b + 2] - az, pts[3 * c] - ax, pts[3 * c + 1] - ay,
                                          pts[3 * c + 2] - az, alpha2, f))
                    continue;
                double tp = INFINITY, tm = -INFINITY;
                bool blocked = false;
                for (int j : all) {
                    if (j == b || j == c) continue;
                    if (gms_alpha_face_point(f, pts[3 * j] - ax, pts[3 * j + 1] - ay, pts[3 * j + 2] - az, tp, tm, blocked)) break;
                }
                if (!gms_alpha_face_decide(f, tp, tm, blocked)) continue;
                if (F < cap) { faces[3 * F] = a; faces[3 * F + 1] = b; faces[3 * F + 2] = c; }
                F++;
            }
    }
    return F;
}

// the smallest-eigenvalue unit eigenvector of symmetric 3x3 matrices [n,6] (xx xy xz yy yz zz), then oriented along d [n,3]
void shim_min_eigvec(int n, const double* A6, const double* d, double* out) {
    for (int i = 0; i < n; i++) {
        gms_sym3_min_eigvec(A6 + 6 * i, out + 3 * i);
        gms_normal_orient(out + 3 * i, d[3 * i], d[3 * i + 1], d[3 * i + 2]);
    }
}

}  // extern "C"
