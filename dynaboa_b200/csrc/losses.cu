// Camera projection, the adaptation losses and the GMM pose prior, each computed together with its
// gradient (loss heads are scalar sums, so the adjoint is produced in the same pass).
//
// Replaces the ATen op chains behind reference base_adaptor.py:160-170 (projection),
// :234-241/:283-291 (frame losses), :331-337 (teacher consistency), :360-370 (labelled exemplar
// losses), :387-396 (motion loss), :401-409 (priors), :412-422 (hip-centred 3D loss),
// utils/geometry.py:184-306 and utils/smplify/prior.py:181-196 -- SURVEY.md §2.1 K8/K9/K10.
#include "common.cuh"
#include "kernels.h"
#include "rotmath.cuh"
#include "losses.h"

namespace dboa {

// ---------------------------------------------------------------------------------------------
// projection: thread per (body, joint)
// ---------------------------------------------------------------------------------------------
__global__ void project_fwd_kernel(const float* __restrict__ cam, const float* __restrict__ j3d, float* __restrict__ p2d, int B, int NJ) {
    pdl_wait();
    pdl_trigger();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * NJ) return;
    int b = i / NJ;
    float c[3] = {cam[b * 3], cam[b * 3 + 1], cam[b * 3 + 2]}, X[3] = {j3d[(size_t)i * 3], j3d[(size_t)i * 3 + 1], j3d[(size_t)i * 3 + 2]}, p[2];
    project_fwd(c, X, p);
    p2d[(size_t)i * 2] = p[0]; p2d[(size_t)i * 2 + 1] = p[1];
}
// one warp per body; dj3d (+)= , dcam (+)=
__global__ void project_bwd_kernel(const float* __restrict__ cam, const float* __restrict__ j3d, const float* __restrict__ dp2d,
                                   float* __restrict__ dj3d, float* __restrict__ dcam, int NJ, int acc_j, int acc_c) {
    pdl_wait();
    pdl_trigger();
    const int b = blockIdx.x, lane = threadIdx.x;
    float c[3] = {cam[b * 3], cam[b * 3 + 1], cam[b * 3 + 2]};
    float dc[3] = {0.f, 0.f, 0.f};
    for (int j = lane; j < NJ; j += 32) {
        size_t i = (size_t)b * NJ + j;
        float X[3] = {j3d[i * 3], j3d[i * 3 + 1], j3d[i * 3 + 2]}, dp[2] = {dp2d[i * 2], dp2d[i * 2 + 1]};
        float dX[3] = {0.f, 0.f, 0.f};
        project_bwd(c, X, dp, dX, dc);
        for (int k = 0; k < 3; ++k) dj3d[i * 3 + k] = acc_j ? dj3d[i * 3 + k] + dX[k] : dX[k];
    }
    for (int k = 0; k < 3; ++k) dc[k] = warp_sum(dc[k]);
    if (lane == 0)
        for (int k = 0; k < 3; ++k) dcam[b * 3 + k] = acc_c ? dcam[b * 3 + k] + dc[k] : dc[k];
}
int project_fwd_launch(const float* cam, const float* j3d, float* p2d, int B, int NJ, cudaStream_t st) {
    return launch_ex(project_fwd_kernel, dim3(ceil_div(B * NJ, 128)), dim3(128), 0, st, dim3(1, 1, 1), true, cam, j3d, p2d, B, NJ);
}
int project_bwd_launch(const float* cam, const float* j3d, const float* dp2d, float* dj3d, float* dcam, int B, int NJ, int acc_j, int acc_c,
                       cudaStream_t st) {
    return launch_ex(project_bwd_kernel, dim3(B), dim3(32), 0, st, dim3(1, 1, 1), true, cam, j3d, dp2d, dj3d, dcam, NJ, acc_j, acc_c);
}

// ---------------------------------------------------------------------------------------------
// pose prior: one 256-thread block per body, warp m evaluates mixture component m
// ---------------------------------------------------------------------------------------------
// FROM_ROT: input is the (24,3,3) rotation stack, gradient goes to d_rot (B,24,3,3)
// otherwise : input is the 69-d axis-angle body pose, gradient goes to d_in (B,69)
template <bool FROM_ROT>
__global__ void __launch_bounds__(256) pose_prior_kernel(const float* __restrict__ in, const float* __restrict__ means,
                                                         const float* __restrict__ prec, const float* __restrict__ neg_log_w,
                                                         float* __restrict__ prior_b, float* __restrict__ d_in, float scale) {
    pdl_wait();
    pdl_trigger();
    __shared__ float sx[69], sd[8][69], sPd[8][69], sg[8][69], sll[8];
    __shared__ int sbest;
    const int b = blockIdx.x, t = threadIdx.x, m = t >> 5, lane = t & 31;
    if (FROM_ROT) {
        if (t < 23) {
            float R[9], aa[3];
            for (int k = 0; k < 9; ++k) R[k] = in[(size_t)b * 216 + (t + 1) * 9 + k];
            r2aa_fwd(R, aa);
            sx[t * 3] = aa[0]; sx[t * 3 + 1] = aa[1]; sx[t * 3 + 2] = aa[2];
        }
    } else {
        if (t < 69) sx[t] = in[(size_t)b * 69 + t];
    }
    __syncthreads();
    for (int c = lane; c < 69; c += 32) sd[m][c] = sx[c] - means[m * 69 + c];
    __syncwarp();
    // pass 1 (one warp per Gaussian): P^T d by columns -- coalesced rows, no shuffles inside the loop, 8 rows in flight;
    // d^T P d = d . (P^T d).  The row products P d are only needed for the gradient of the selected component (pass 2).
    float accT[3] = {0.f, 0.f, 0.f};
    const float* P = prec + (size_t)m * 69 * 69;
#pragma unroll 8
    for (int i = 0; i < 69; ++i) {
        const float di = sd[m][i];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const int c = lane + q * 32;
            if (c < 69) accT[q] = fmaf(di, __ldg(P + i * 69 + c), accT[q]);
        }
    }
    float quad = 0.f;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const int c = lane + q * 32;
        if (c < 69) { quad = fmaf(sd[m][c], accT[q], quad); sg[m][c] = accT[q]; }
    }
    quad = warp_sum(quad);
    if (lane == 0) sll[m] = 0.5f * quad + neg_log_w[m];
    __syncthreads();
    if (t == 0) {
        int best = 0;
        for (int k = 1; k < 8; ++k)
            if (sll[k] < sll[best]) best = k;
        sbest = best;
        prior_b[b] = sll[best];
    }
    __syncthreads();
    if (d_in != nullptr) {                                     // pass 2: rows of the selected precision matrix, 8 warps x 9 rows
        const int k = sbest;
        const float* Pk = prec + (size_t)k * 69 * 69;
        for (int i = m; i < 69; i += 8) {
            float rowdot = 0.f;
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const int c = lane + q * 32;
                if (c < 69) rowdot = fmaf(__ldg(Pk + i * 69 + c), sd[k][c], rowdot);
            }
            rowdot = warp_sum(rowdot);
            if (lane == 0) sPd[0][i] = 0.5f * (rowdot + sg[k][i]);     // d(0.5 d^T P d) = 0.5 (P + P^T) d
        }
    }
    __syncthreads();
    if (d_in != nullptr) {
        if (FROM_ROT) {
            if (t < 9) d_in[(size_t)b * 216 + t] = 0.f;            // root joint carries no prior
            if (t < 23) {
                float R[9], daa[3], dR[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                for (int k = 0; k < 9; ++k) R[k] = in[(size_t)b * 216 + (t + 1) * 9 + k];
                for (int k = 0; k < 3; ++k) daa[k] = sPd[0][t * 3 + k] * scale;
                r2aa_bwd(R, daa, dR);
                for (int k = 0; k < 9; ++k) d_in[(size_t)b * 216 + (t + 1) * 9 + k] = dR[k];
            }
        } else {
            if (t < 69) d_in[(size_t)b * 69 + t] = sPd[0][t] * scale;
        }
    }
}
int pose_prior_launch(const float* rot, const float* means, const float* prec, const float* neg_log_w, float* prior_b, float* drot,
                      float scale, int B, cudaStream_t st) {
    return launch_ex(pose_prior_kernel<true>, dim3(B), dim3(256), 0, st, dim3(1, 1, 1), true, rot, means, prec, neg_log_w, prior_b, drot, scale);
}
int gmm_prior_launch(const float* pose69, const float* means, const float* prec, const float* neg_log_w, float* prior_b, float* dpose,
                     float scale, int B, cudaStream_t st) {
    return launch_ex(pose_prior_kernel<false>, dim3(B), dim3(256), 0, st, dim3(1, 1, 1), true, pose69, means, prec, neg_log_w, prior_b, dpose, scale);
}

// ---------------------------------------------------------------------------------------------
// multi-term loss head: a single 256-thread block covers the (small) batch
// terms: 0 s2d(masked, joints 25..48)  1 shape prior  2 pose prior (value only, from prior_b)
//        3 target p2d MSE  4 target j3d MSE  5 target beta MSE  6 target R MSE  7 hip-centred 3D
// ---------------------------------------------------------------------------------------------
// grouped (a.groups > 1): block g computes video g's terms on its own rows
__global__ void __launch_bounds__(256) loss_multi_kernel(LossArgs a) {
    pdl_wait();
    pdl_trigger();
    __shared__ float red[32];
    __shared__ float sterm[8];
    const int B = a.B / gridDim.x;
    if (gridDim.x > 1) {
        const size_t r = (size_t)blockIdx.x * B;
        auto off = [&](auto& p, size_t per_row) { if (p != nullptr) p += r * per_row; };
        off(a.p2d, 98); off(a.j3d, 147); off(a.R, 216); off(a.beta, 10); off(a.kp, 147); off(a.prior_b, 1); off(a.t_p2d, 98);
        off(a.t_j3d, 147); off(a.t_beta, 10); off(a.t_R, 216); off(a.gt_s3d, 96); off(a.dp2d, 98); off(a.dj3d, 147); off(a.dR, 216);
        off(a.dbeta, 10);
        a.terms += 9 * blockIdx.x;
    }
    const int t = threadIdx.x;
    const int kf = a.kp_count > 0 ? a.kp_first : 25, kn = a.kp_count > 0 ? a.kp_count : 24;      // joints of the re-projection term
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};

    // ---- 2D terms over (b, joint, xy)
    for (int i = t; i < B * 49 * 2; i += 256) {
        const int j = (i / 2) % 49, b = i / 98;
        const float p = a.p2d[i];
        float g = 0.f;
        if (a.kp != nullptr && j >= kf && j < kf + kn) {
            const float conf = a.kp[(size_t)(b * 49 + j) * 3 + 2];
            const float k = a.kp[(size_t)(b * 49 + j) * 3 + (i & 1)];
            const float d = p - k;
            acc[0] += d * d * conf;
            g += a.w[0] * 2.0f * conf * d / (float)(B * kn * 2);
        }
        if (a.t_p2d != nullptr) {
            const float d = p - a.t_p2d[i];
            acc[3] += d * d;
            g += a.w[3] * 2.0f * d / (float)(B * 98);
        }
        if (a.dp2d != nullptr) a.dp2d[i] = g;
    }
    // ---- 3D target term over (b, joint, xyz); the hip-centred labelled term is added below
    for (int i = t; i < B * 147; i += 256) {
        float g = 0.f;
        if (a.t_j3d != nullptr) {
            const float d = a.j3d[i] - a.t_j3d[i];
            acc[4] += d * d;
            g = a.w[4] * 2.0f * d / (float)(B * 147);
        }
        if (a.dj3d != nullptr) a.dj3d[i] = g;
    }
    // ---- shape terms
    for (int i = t; i < B * 10; i += 256) {
        const float be = a.beta[i];
        acc[1] += be * be;
        float g = a.w[1] * 2.0f * be / (float)B;
        if (a.t_beta != nullptr) {
            const float d = be - a.t_beta[i];
            acc[5] += d * d;
            g += a.w[5] * 2.0f * d / (float)(B * 10);
        }
        if (a.dbeta != nullptr) a.dbeta[i] = g;
    }
    // ---- rotation target term (dR may already hold the pose-prior gradient)
    for (int i = t; i < B * 216; i += 256) {
        float g = 0.f;
        if (a.t_R != nullptr) {
            const float d = a.R[i] - a.t_R[i];
            acc[6] += d * d;
            g = a.w[6] * 2.0f * d / (float)(B * 216);
        }
        if (a.dR != nullptr) a.dR[i] = a.dR_accumulate ? a.dR[i] + g : g;
    }
    __syncthreads();
    // ---- hip-centred 3D loss on the 24 ground-truth joints (49-joint indices 25..48), thread per body
    if (a.gt_s3d != nullptr && t < B) {
        const int b = t;
        const float* pj = a.j3d + (size_t)b * 147 + 25 * 3;
        const float* gj = a.gt_s3d + (size_t)b * 96;
        float ph[3], gh[3], sum_e[3] = {0.f, 0.f, 0.f};
        for (int k = 0; k < 3; ++k) { ph[k] = (pj[2 * 3 + k] + pj[3 * 3 + k]) / 2.0f; gh[k] = (gj[2 * 4 + k] + gj[3 * 4 + k]) / 2.0f; }
        const float gs = a.w[7] * 2.0f / (float)(B * 72);
        for (int j = 0; j < 24; ++j) {
            const float conf = a.kp[(size_t)(b * 49 + 25 + j) * 3 + 2];
            for (int k = 0; k < 3; ++k) {
                const float d = (pj[j * 3 + k] - ph[k]) - (gj[j * 4 + k] - gh[k]);
                acc[7] += conf * d * d;
                const float e = gs * conf * d;
                sum_e[k] += e;
                if (a.dj3d != nullptr) a.dj3d[(size_t)b * 147 + (25 + j) * 3 + k] += e;
            }
        }
        if (a.dj3d != nullptr)
            for (int k = 0; k < 3; ++k) {
                a.dj3d[(size_t)b * 147 + 27 * 3 + k] -= 0.5f * sum_e[k];
                a.dj3d[(size_t)b * 147 + 28 * 3 + k] -= 0.5f * sum_e[k];
            }
    }
    // ---- scalar terms
    const float norm[8] = {1.0f / (B * kn * 2), 1.0f / B, 1.0f, 1.0f / (B * 98), 1.0f / (B * 147), 1.0f / (B * 10), 1.0f / (B * 216),
                           1.0f / (B * 72)};
    for (int k = 0; k < 8; ++k) {
        float s = block_sum(acc[k], red);
        if (t == 0) sterm[k] = s * norm[k];
    }
    if (t == 0) {
        if (a.prior_b != nullptr) {
            float s = 0.f;
            for (int b = 0; b < B; ++b) s += a.prior_b[b];
            sterm[2] = s / (float)B;
        } else sterm[2] = 0.f;
        float total = 0.f;
        for (int k = 0; k < 8; ++k) { a.terms[k] = sterm[k]; total += a.w[k] * sterm[k]; }
        a.terms[8] = total;
    }
}
int loss_multi_launch(const LossArgs& a, cudaStream_t st) {
    const int groups = a.groups > 1 ? a.groups : 1;
    if (a.B < 1 || a.B > 256 * groups || a.groups < 0 || a.B % groups != 0) return DBOA_ERR_SHAPE;
    if (a.kp_count < 0 || a.kp_first < 0 || a.kp_first + a.kp_count > 49) return DBOA_ERR_ARG;
    return launch_ex(loss_multi_kernel, dim3(groups), dim3(256), 0, st, dim3(1, 1, 1), true, a);
}

// ---------------------------------------------------------------------------------------------
// motion loss between the current prediction (a) and the prediction on the history frame (h)
//   L = mean_{B*count*2} [conf_a + conf_h == 2] * ((pa - ph) - (ka - kh))^2   on joints [first, first + count)  (benchmark: 25..48)
// A video whose `active` bit is clear gets term 0 and leaves its rows of dpa and dph untouched.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) loss_motion_kernel(const float* __restrict__ pa, const float* __restrict__ ph,
                                                          const float* __restrict__ ka, const float* __restrict__ kh, float w,
                                                          float* __restrict__ term, float* __restrict__ dpa, float* __restrict__ dph,
                                                          int B, int acc_a, int first, int count, unsigned long long active) {
    pdl_wait();
    pdl_trigger();
    __shared__ float red[32];
    B /= gridDim.x;                                          // grouped: block g takes video g's B rows
    if (blockIdx.x < 64 && !((active >> blockIdx.x) & 1ULL)) {
        if (threadIdx.x == 0) term[blockIdx.x] = 0.f;
        return;
    }
    {
        const size_t r = (size_t)blockIdx.x * B;
        pa += r * 98; ph += r * 98; ka += r * 147; kh += r * 147; dpa += r * 98; dph += r * 98; term += blockIdx.x;
    }
    float acc = 0.f;
    const float n = (float)(B * count * 2);
    for (int i = threadIdx.x; i < B * 98; i += 256) {
        const int j = (i / 2) % 49, b = i / 98;
        float g = 0.f;
        if (j >= first && j < first + count) {
            const size_t kb = (size_t)(b * 49 + j) * 3;
            const float conf = (ka[kb + 2] + kh[kb + 2]) == 2.0f ? 1.0f : 0.0f;
            const float d = (pa[i] - ph[i]) - (ka[kb + (i & 1)] - kh[kb + (i & 1)]);
            acc += conf * d * d;
            g = w * 2.0f * conf * d / n;
        }
        dpa[i] = acc_a ? dpa[i] + g : g;
        dph[i] = -g;
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) term[0] = acc / n;
}
int loss_motion_launch(const float* pa, const float* ph, const float* ka, const float* kh, float w, float* term, float* dpa, float* dph,
                       int B, int acc_a, int first, int count, cudaStream_t st, int groups, unsigned long long active) {
    if (first < 0 || count < 1 || first + count > 49) return DBOA_ERR_ARG;
    if (groups < 1 || B % groups != 0) return DBOA_ERR_SHAPE;
    return launch_ex(loss_motion_kernel, dim3(groups), dim3(256), 0, st, dim3(1, 1, 1), true, pa, ph, ka, kh, w, term, dpa, dph, B, acc_a, first,
                     count, active);
}

}  // namespace dboa
