// Evaluation metrics of one adapted frame on the device: H36M-regressor joints, MPJPE, Procrustes-aligned MPJPE
// (PA-MPJPE) and per-vertex error (PVE).
//
// Replaces reference dynaboa_benchmark.py:217-240 (Adaptor.inference: two dense J_regressor products, the pelvis
// centring / 14-joint selection, `compute_similarity_transform_batch` -- utils/pose_utils.py:9-64, a per-sample numpy
// SVD after a device->host copy of the joints -- and the PVE, computed on the host from 2 x 6890 x 3 floats).
// SURVEY.md section 8f row N1.  The whole evaluation becomes two launches and ONE 3-float read-back per sample.
//
//   launch 1, grid (NJ, B, 3): z = 0 / 1: joint j of the predicted / ground-truth mesh = sum_v Jreg[j][v] * verts[b][v][:]
//                              z = 2    : partial sum of |gt_neutral - pred| over the j-th slice of the vertices
//   launch 2, one thread per sample (fp64): centre on joint 0, pick the 14 evaluation joints, MPJPE, similarity
//             Procrustes with a one-sided Jacobi SVD of the 3x3 covariance, PA-MPJPE, PVE = sum of the partials / V.
// Orientation fix as in the reference: R = V diag(1, 1, sign(det(U V^T))) U^T with the sign on the SMALLEST singular value
// (numpy returns singular values sorted, so its last column is the smallest).
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace dboa {

constexpr int EV_NT = 256;
constexpr int EV_MAXJ = 32;

__global__ void __launch_bounds__(EV_NT) eval_joints_kernel(const float* __restrict__ pred, const float* __restrict__ gt_j,
                                                            const float* __restrict__ gt_v, const float* __restrict__ Jreg, int NV,
                                                            float* __restrict__ scratch /* [B][2][NJ][3] joints, then [B][NJ] pve partials */,
                                                            int per_video, unsigned long long active) {
    __shared__ float red[32];
    const int j = blockIdx.x, b = blockIdx.y, z = blockIdx.z, NJ = gridDim.x, B = gridDim.y;
    if (!((active >> (b / per_video)) & 1ULL)) return;                // idle video: uniform over the CTA, before the wait
    pdl_wait();
    pdl_trigger();
    if (z < 2) {
        const float* v = (z == 0 ? pred : gt_j) + (size_t)b * NV * 3;
        const float* w = Jreg + (size_t)j * NV;
        float ax = 0.f, ay = 0.f, az = 0.f;
        for (int i = threadIdx.x; i < NV; i += EV_NT) {
            const float wi = __ldg(w + i);
            ax = fmaf(wi, __ldg(v + i * 3), ax); ay = fmaf(wi, __ldg(v + i * 3 + 1), ay); az = fmaf(wi, __ldg(v + i * 3 + 2), az);
        }
        ax = block_sum(ax, red); ay = block_sum(ay, red); az = block_sum(az, red);
        if (threadIdx.x == 0) {
            float* o = scratch + (((size_t)b * 2 + z) * NJ + j) * 3;
            o[0] = ax; o[1] = ay; o[2] = az;
        }
    } else {
        const int per = (NV + NJ - 1) / NJ, v0 = j * per, v1 = min(NV, v0 + per);
        const float* p = pred + (size_t)b * NV * 3;
        const float* g = gt_v + (size_t)b * NV * 3;
        float s = 0.f;
        for (int i = v0 + threadIdx.x; i < v1; i += EV_NT) {
            const float dx = __ldg(g + i * 3) - __ldg(p + i * 3), dy = __ldg(g + i * 3 + 1) - __ldg(p + i * 3 + 1),
                        dz = __ldg(g + i * 3 + 2) - __ldg(p + i * 3 + 2);
            s += sqrtf(dx * dx + dy * dy + dz * dz);
        }
        s = block_sum(s, red);
        if (threadIdx.x == 0) scratch[(size_t)B * 2 * NJ * 3 + (size_t)b * NJ + j] = s;
    }
}

// one-sided (Hestenes) Jacobi SVD of a 3x3 matrix: A V = U S.  a: in A (row-major), out the orthogonalised columns U S.
__device__ void svd3_jacobi(double a[3][3], double v[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) v[i][k] = i == k ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                double alpha = 0.0, beta = 0.0, gamma = 0.0;
                for (int i = 0; i < 3; ++i) { alpha += a[i][p] * a[i][p]; beta += a[i][q] * a[i][q]; gamma += a[i][p] * a[i][q]; }
                if (fabs(gamma) <= 1e-300 || fabs(gamma) <= 1e-15 * sqrt(alpha * beta)) continue;
                off = fmax(off, fabs(gamma) / sqrt(alpha * beta));
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int i = 0; i < 3; ++i) {
                    const double ap = a[i][p], aq = a[i][q];
                    a[i][p] = c * ap - s * aq; a[i][q] = s * ap + c * aq;
                    const double vp = v[i][p], vq = v[i][q];
                    v[i][p] = c * vp - s * vq; v[i][q] = s * vp + c * vq;
                }
            }
        if (off < 1e-14) break;
    }
}

__global__ void eval_metrics_kernel(const float* __restrict__ scratch, const int* __restrict__ joint_map, int n_map, int NJ, int NV, int B,
                                    float* __restrict__ out /* [B][3]: mpjpe, pa-mpjpe, pve */, int per_video, unsigned long long active) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B || !((active >> (b / per_video)) & 1ULL)) return;       // idle rows exit before the wait
    pdl_wait();
    pdl_trigger();
    const float* jp = scratch + ((size_t)b * 2 + 0) * NJ * 3;
    const float* jg = scratch + ((size_t)b * 2 + 1) * NJ * 3;
    double S1[EV_MAXJ][3], S2[EV_MAXJ][3];
    double mu1[3] = {0, 0, 0}, mu2[3] = {0, 0, 0}, mpjpe = 0.0;
    for (int i = 0; i < n_map; ++i) {
        const int j = joint_map[i];
        double d2 = 0.0;
        for (int k = 0; k < 3; ++k) {
            S1[i][k] = (double)jp[j * 3 + k] - (double)jp[k];          // pelvis (regressor joint 0) centred, as the reference
            S2[i][k] = (double)jg[j * 3 + k] - (double)jg[k];
            mu1[k] += S1[i][k]; mu2[k] += S2[i][k];
            const double d = S1[i][k] - S2[i][k];
            d2 += d * d;
        }
        mpjpe += sqrt(d2);
    }
    mpjpe /= n_map;
    for (int k = 0; k < 3; ++k) { mu1[k] /= n_map; mu2[k] /= n_map; }
    // K = X1 X2^T (3x3), var1 = |X1|^2
    double K[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, var1 = 0.0;
    for (int i = 0; i < n_map; ++i)
        for (int r = 0; r < 3; ++r) {
            const double x1 = S1[i][r] - mu1[r];
            var1 += x1 * x1;
            for (int c = 0; c < 3; ++c) K[r][c] += x1 * (S2[i][c] - mu2[c]);
        }
    double a[3][3], V[3][3], U[3][3], sv[3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) a[r][c] = K[r][c];
    svd3_jacobi(a, V);
    int smallest = 0;
    double sv_max = 0.0;
    for (int c = 0; c < 3; ++c) {
        sv[c] = sqrt(a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c]);
        if (sv[c] < sv[smallest]) smallest = c;
        sv_max = fmax(sv_max, sv[c]);
    }
    // U = the normalised non-zero columns, completed to an orthonormal basis for every rank of the covariance: a zero
    // column of U S is any unit vector orthogonal to the others (planar joints give rank 2, collinear ones rank 1,
    // coincident ones 0), so every entry of U is set before R reads it.  A column counts as zero relative to the largest:
    // for an exactly rank-deficient covariance the Jacobi sweeps leave rounding residue in the spare columns, as small as
    // 1e-16 of the largest or down in the range where their squares underflow and the rotations stall, and that residue
    // points along the real columns, not across them
    const double zero_sv = 1e-12 * sv_max;
    int rank = 0, nz = 0;
    for (int c = 0; c < 3; ++c) {
        if (sv[c] > zero_sv) {
            for (int r = 0; r < 3; ++r) U[r][c] = a[r][c] / sv[c];
            ++rank;
            nz = c;
        } else {
            for (int r = 0; r < 3; ++r) U[r][c] = r == c ? 1.0 : 0.0;  // rank 0: the identity
        }
    }
    if (rank == 1) {                                                   // Gram-Schmidt of the least aligned axis against column nz
        const int z = (smallest + 1) % 3 != nz ? (smallest + 1) % 3 : (smallest + 2) % 3;   // the zero column other than smallest
        int k = 0;
        for (int r = 1; r < 3; ++r)
            if (fabs(U[r][nz]) < fabs(U[k][nz])) k = r;
        double e[3] = {0.0, 0.0, 0.0}, len = 0.0;
        for (int r = 0; r < 3; ++r) { e[r] = (r == k ? 1.0 : 0.0) - U[k][nz] * U[r][nz]; len += e[r] * e[r]; }
        len = sqrt(len);
        for (int r = 0; r < 3; ++r) U[r][z] = e[r] / len;
    }
    if (sv[smallest] <= zero_sv) {                                     // rank-deficient covariance: complete U with a cross product
        const int c1 = (smallest + 1) % 3, c2 = (smallest + 2) % 3;
        U[0][smallest] = U[1][c1] * U[2][c2] - U[2][c1] * U[1][c2];
        U[1][smallest] = U[2][c1] * U[0][c2] - U[0][c1] * U[2][c2];
        U[2][smallest] = U[0][c1] * U[1][c2] - U[1][c1] * U[0][c2];
    }
    // det(U V^T) = det(U) det(V)
    auto det3 = [](const double m[3][3]) {
        return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
               m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
    };
    const double dsign = det3(U) * det3(V);
    const double zs = dsign > 0.0 ? 1.0 : (dsign < 0.0 ? -1.0 : 0.0);
    double R[3][3];                                                    // R = V Z U^T
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += V[r][k] * (k == smallest ? zs : 1.0) * U[c][k];
            R[r][c] = s;
        }
    double tr = 0.0;                                                   // trace(R K)
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) tr += R[r][k] * K[k][r];
    const double scale = tr / var1;
    double t[3];
    for (int r = 0; r < 3; ++r) t[r] = mu2[r] - scale * (R[r][0] * mu1[0] + R[r][1] * mu1[1] + R[r][2] * mu1[2]);
    double pa = 0.0;
    for (int i = 0; i < n_map; ++i) {
        double d2 = 0.0;
        for (int r = 0; r < 3; ++r) {
            const double h = scale * (R[r][0] * S1[i][0] + R[r][1] * S1[i][1] + R[r][2] * S1[i][2]) + t[r];
            d2 += (h - S2[i][r]) * (h - S2[i][r]);
        }
        pa += sqrt(d2);
    }
    pa /= n_map;
    double pve = 0.0;
    const float* part = scratch + (size_t)B * 2 * NJ * 3 + (size_t)b * NJ;
    for (int j = 0; j < NJ; ++j) pve += (double)part[j];
    out[b * 3 + 0] = (float)mpjpe; out[b * 3 + 1] = (float)pa; out[b * 3 + 2] = (float)(pve / NV);
}

size_t eval_scratch_floats(int B, int NJ) { return (size_t)B * 2 * NJ * 3 + (size_t)B * NJ; }

// `groups` videos of B / groups rows each; only the rows of the videos whose bit is set in `active` are read, computed and
// written.  A row's arithmetic does not depend on the other rows, so an active row is bit-identical to a call on its rows alone.
int eval_metrics(const float* pred_verts, const float* gt_verts_joints, const float* gt_verts_pve, const float* Jreg, int NJ, int NV,
                 const int* joint_map, int n_map, float* scratch, float* out, int B, int groups, unsigned long long active, cudaStream_t st) {
    if (NJ < 1 || NJ > EV_MAXJ || n_map < 1 || n_map > EV_MAXJ || B < 1) return DBOA_ERR_SHAPE;
    if (groups < 1 || groups > 64 || B % groups != 0) return DBOA_ERR_SHAPE;
    if (active == 0 || (groups < 64 && (active >> groups) != 0)) return DBOA_ERR_ARG;
    const int per_video = B / groups;
    DBOA_TRY(launch_ex(eval_joints_kernel, dim3(NJ, B, 3), dim3(EV_NT), 0, st, dim3(1, 1, 1), true, pred_verts, gt_verts_joints, gt_verts_pve,
                       Jreg, NV, scratch, per_video, active));
    return launch_ex(eval_metrics_kernel, dim3(ceil_div(B, 64)), dim3(64), 0, st, dim3(1, 1, 1), true, (const float*)scratch, joint_map, n_map,
                     NJ, NV, B, out, per_video, active);
}

}  // namespace dboa
