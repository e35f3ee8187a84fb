// Mesh overlay: one mesh drawn over one 8-bit frame, entirely on the device.
//
// Replaces reference render_demo.py:58-153 (Renderer.render: trimesh + pyrender off-screen OpenGL, 4x multisampled, read back
// and composited with numpy) as called by base_adaptor.py:429-443 (save_results) and utils/webcam_utils.py:71-79 (render).
// The contract is DESIGN.md section 6 "Mesh overlay"; in short:
//
//   render frame   p' = A . Rx(180) . v               (:88-98; A = optional angle/axis rotation, Rx(x,y,z) = (x,-y,-z))
//   window         u = (1 + sx (p'x + tx)) / 2 * W,  r = (1 - sy (p'y - ty)) / 2 * H,  ndc_z = -p'z
//                  (WeakPerspectiveCamera :48-55 with pyrender's vertical flip of the read-back; row 0 = top)
//   raster         window coordinates snapped to 1/256 pixel, int64 edge functions, top-left fill rule in image
//                  coordinates (rows down); faces with a vertex beyond +-2^20 pixels are dropped (guard band);
//                  drawn iff (b - a) x (c - a) < 0 in image coordinates (GL_CULL_FACE / GL_BACK); fragments with
//                  ndc_z outside [-1, 1] are discarded (near / far planes); smaller ndc_z wins, then the lower face id
//   depth          ((e0 z0 + e1 z1) + e2 z2) / A in double without contraction, rounded to fp32
//   samples        1 (pixel centre) or 4 (offsets (-2,-6) (6,-2) (-6,2) (2,6) / 16 pixel from the centre)
//   shading        pyrender's metallic-roughness shader at metallic 0, roughness 1, ambient 0.3 and three white point
//                  lights at (0,-1,1), (0,1,1), (1,1,2) (:72-84), once per (pixel, face) at the pixel centre, with trimesh's
//                  angle-weighted vertex normals; UNPINNED restatement (pyrender / trimesh / EGL are not available here)
//   composite      each sample's byte round(255 c), uncovered samples black; pixel = rounded mean over the samples when
//                  at least one is covered (:126-129), else the input pixel unchanged
//
// Launches (no host round trip): vertex transform -> vertex normals (vertex->face CSR, fixed summation order, no float
// atomics) -> face set-up (cull, bounding box, number of 8x8 pixel tiles) -> prefix sum of the tile counts -> clear the
// depth keys -> raster, one warp per (face, tile) pair, keeps min(key) per sample with a 64-bit integer atomicMin on
// key = order-preserving fp32 depth bits << 32 | face id (the result does not depend on launch order) -> resolve, one
// thread per pixel.  Everything geometric is computed in double or integers, so the oracle (oracle/render_ref.py, numpy
// float64) reproduces every winning face bit for bit.
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace dboa {

namespace {

constexpr int RT = 8;                              // raster tile: 8 x 8 pixels per (face, tile) pair
constexpr double GUARD = 1048576.0;                // 2^20 pixels
constexpr unsigned long long EMPTY = ~0ull;

struct RenderCam {
    double sx, sy, tx, ty;
    double R[9];
    int has_rot;
    int W, H, S;
};

struct Scratch {
    double* pr;                  // [NV][3] render-frame positions
    double* nrm;                 // [NV][3] vertex normals
    long long* fx;               // [NV][2] window position, 24.8 fixed point
    double* vz;                  // [NV]    ndc_z
    int* vok;                    // [NV]    inside the guard band
    int4* fidx;                  // [NF]    vertex indices in raster order (a, c, b), w = 0
    int4* fbox;                  // [NF]    pixel box c0, r0, c1, r1
    long long* prefix;           // [NF + 1] exclusive prefix sum of the tile counts (entry NF = number of pairs)
    unsigned long long* keys;    // [H][W][S]
};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t carve(Scratch* s, char* base, int W, int H, int NV, int NF, int S) {
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
    char* pr = take((size_t)NV * 3 * sizeof(double));
    char* nrm = take((size_t)NV * 3 * sizeof(double));
    char* fx = take((size_t)NV * 2 * sizeof(long long));
    char* vz = take((size_t)NV * sizeof(double));
    char* vok = take((size_t)NV * sizeof(int));
    char* fidx = take((size_t)NF * sizeof(int4));
    char* fbox = take((size_t)NF * sizeof(int4));
    char* prefix = take(((size_t)NF + 1) * sizeof(long long));
    char* keys = take((size_t)W * H * S * sizeof(unsigned long long));
    if (s) {
        s->pr = (double*)pr; s->nrm = (double*)nrm; s->fx = (long long*)fx; s->vz = (double*)vz; s->vok = (int*)vok;
        s->fidx = (int4*)fidx; s->fbox = (int4*)fbox; s->prefix = (long long*)prefix; s->keys = (unsigned long long*)keys;
    }
    return off;
}

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dadd_rn(a, -b); }

__global__ void render_vertex_kernel(const float* __restrict__ verts, int NV, RenderCam c, Scratch s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NV) return;
    const size_t i3 = (size_t)i * 3;
    const double q[3] = {(double)verts[i3], -(double)verts[i3 + 1], -(double)verts[i3 + 2]};
    double p[3] = {q[0], q[1], q[2]};
    if (c.has_rot)
        for (int k = 0; k < 3; ++k) p[k] = da(da(dm(c.R[k * 3], q[0]), dm(c.R[k * 3 + 1], q[1])), dm(c.R[k * 3 + 2], q[2]));
    const double u = dm(dm(da(1.0, dm(c.sx, da(p[0], c.tx))), 0.5), (double)c.W);
    const double r = dm(dm(ds(1.0, dm(c.sy, ds(p[1], c.ty))), 0.5), (double)c.H);
    const bool ok = fabs(u) <= GUARD && fabs(r) <= GUARD;            // false for NaN as well
    for (int k = 0; k < 3; ++k) s.pr[i3 + k] = p[k];
    s.fx[(size_t)i * 2] = ok ? __double2ll_rn(u * 256.0) : 0;
    s.fx[(size_t)i * 2 + 1] = ok ? __double2ll_rn(r * 256.0) : 0;
    s.vz[i] = -p[2];
    s.vok[i] = ok;
}

// trimesh Trimesh.vertex_normals: sum over the incident faces of (corner angle) * (unit face normal), normalised.  Faces with
// zero area contribute nothing; a corner angle below 1e-8 zeroes all three angles of its face (triangles.angles).
__global__ void render_normal_kernel(const int* __restrict__ faces, int NF, int NV, const int* __restrict__ vf_off,
                                     const int* __restrict__ vf_faces, Scratch s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NV) return;
    double acc[3] = {0.0, 0.0, 0.0};
    for (int e = vf_off[i]; e < vf_off[i + 1]; ++e) {
        const int f = vf_faces[e];
        if (f < 0 || f >= NF) continue;
        int id[3], corner = -1;
        bool bad = false;
        for (int k = 0; k < 3; ++k) {
            id[k] = faces[(size_t)f * 3 + k];
            bad |= id[k] < 0 || id[k] >= NV;
            if (corner < 0 && id[k] == i) corner = k;
        }
        if (bad || corner < 0) continue;
        double P[3][3];
        for (int k = 0; k < 3; ++k)
            for (int j = 0; j < 3; ++j) P[k][j] = s.pr[id[k] * 3 + j];
        double u[3], v[3], w[3];
        for (int j = 0; j < 3; ++j) { u[j] = ds(P[1][j], P[0][j]); v[j] = ds(P[2][j], P[0][j]); w[j] = ds(P[2][j], P[1][j]); }
        const double n[3] = {ds(dm(u[1], v[2]), dm(u[2], v[1])), ds(dm(u[2], v[0]), dm(u[0], v[2])), ds(dm(u[0], v[1]), dm(u[1], v[0]))};
        const double nn = sqrt(da(da(dm(n[0], n[0]), dm(n[1], n[1])), dm(n[2], n[2])));
        if (!(nn > 0.0)) continue;
        const double lu = sqrt(da(da(dm(u[0], u[0]), dm(u[1], u[1])), dm(u[2], u[2])));
        const double lv = sqrt(da(da(dm(v[0], v[0]), dm(v[1], v[1])), dm(v[2], v[2])));
        const double lw = sqrt(da(da(dm(w[0], w[0]), dm(w[1], w[1])), dm(w[2], w[2])));
        for (int j = 0; j < 3; ++j) { u[j] /= lu; v[j] /= lv; w[j] /= lw; }
        const double a0 = acos(fmin(fmax(da(da(dm(u[0], v[0]), dm(u[1], v[1])), dm(u[2], v[2])), -1.0), 1.0));
        const double a1 = acos(fmin(fmax(-da(da(dm(u[0], w[0]), dm(u[1], w[1])), dm(u[2], w[2])), -1.0), 1.0));
        const double a2 = ds(ds(M_PI, a0), a1);
        if (a0 < 1e-8 || a1 < 1e-8 || a2 < 1e-8) continue;
        const double a = corner == 0 ? a0 : corner == 1 ? a1 : a2;
        for (int j = 0; j < 3; ++j) acc[j] = da(acc[j], dm(a, n[j] / nn));
    }
    const double l = sqrt(da(da(dm(acc[0], acc[0]), dm(acc[1], acc[1])), dm(acc[2], acc[2])));
    for (int j = 0; j < 3; ++j) s.nrm[i * 3 + j] = l > 0.0 ? acc[j] / l : 0.0;
}

__device__ __forceinline__ long long floordiv(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// cull + bounding box; writes the face's tile count to prefix[f + 1]
__global__ void render_face_kernel(const int* __restrict__ faces, int NF, int NV, Scratch s, int W, int H) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= NF) return;
    long long count = 0;
    const int i0 = faces[(size_t)f * 3], i1 = faces[(size_t)f * 3 + 1], i2 = faces[(size_t)f * 3 + 2];
    if (i0 >= 0 && i0 < NV && i1 >= 0 && i1 < NV && i2 >= 0 && i2 < NV && s.vok[i0] && s.vok[i1] && s.vok[i2]) {
        const long long ax = s.fx[i0 * 2], ay = s.fx[i0 * 2 + 1], bx = s.fx[i1 * 2], by = s.fx[i1 * 2 + 1];
        const long long cx = s.fx[i2 * 2], cy = s.fx[i2 * 2 + 1];
        const long long area = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
        if (area < 0) {
            // samples of pixel c lie in [256 c + 32, 256 c + 224] (4x pattern; the centre 256 c + 128 for 1x)
            const long long x0 = min(ax, min(bx, cx)), x1 = max(ax, max(bx, cx));
            const long long y0 = min(ay, min(by, cy)), y1 = max(ay, max(by, cy));
            const long long c0 = max(0ll, -floordiv(-(x0 - 224), 256)), c1 = min((long long)W - 1, floordiv(x1 - 32, 256));
            const long long r0 = max(0ll, -floordiv(-(y0 - 224), 256)), r1 = min((long long)H - 1, floordiv(y1 - 32, 256));
            if (c0 <= c1 && r0 <= r1) {
                count = ((c1 - c0) / RT + 1) * ((r1 - r0) / RT + 1);
                s.fidx[f] = make_int4(i0, i2, i1, 0);             // (a, c, b): positive area in image coordinates
                s.fbox[f] = make_int4((int)c0, (int)r0, (int)c1, (int)r1);
            }
        }
    }
    s.prefix[f + 1] = count;
}

// in-place inclusive scan of prefix[1..NF] by one block (the face count is small; this runs once per draw)
__global__ void __launch_bounds__(1024) render_scan_kernel(long long* __restrict__ prefix, int NF) {
    __shared__ long long warp_tot[32];
    __shared__ long long carry;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry = 0; prefix[0] = 0; }
    __syncthreads();
    for (long long base = 0; base < NF; base += 1024) {
        const long long i = base + threadIdx.x;
        long long v = i < NF ? prefix[i + 1] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const long long t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += t;
        }
        if (lane == 31) warp_tot[wid] = v;
        __syncthreads();
        if (wid == 0) {
            long long t = warp_tot[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const long long u = __shfl_up_sync(0xffffffffu, t, o);
                if (lane >= o) t += u;
            }
            warp_tot[lane] = t;
        }
        __syncthreads();
        const long long c = carry;
        if (i < NF) prefix[i + 1] = c + v + (wid > 0 ? warp_tot[wid - 1] : 0);
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + warp_tot[31];
        __syncthreads();
    }
}

__device__ __forceinline__ long long edge(long long px, long long py, long long qx, long long qy, long long sx, long long sy) {
    return (qx - px) * (sy - py) - (qy - py) * (sx - px);
}
__device__ __forceinline__ bool top_left(long long px, long long py, long long qx, long long qy) {
    return qy < py || (qy == py && qx > px);
}

__constant__ int c_off4[4][2] = {{-32, -96}, {96, -32}, {-96, 32}, {32, 96}};   // 1/256 pixel: (-2,-6) (6,-2) (-6,2) (2,6) / 16

__global__ void __launch_bounds__(256) render_raster_kernel(int NF, Scratch s, int W, int S) {
    const long long total = s.prefix[NF];
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long pair = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; pair < total; pair += nwarps) {
        int lo = 0, hi = NF;                                           // last face with prefix[f] <= pair
        while (lo < hi) {
            const int mid = (int)(((long long)lo + hi + 1) >> 1);
            if (s.prefix[mid] <= pair) lo = mid; else hi = mid - 1;
        }
        const int f = lo;
        const int4 id = s.fidx[f], box = s.fbox[f];
        const long long t = pair - s.prefix[f];
        const int ntx = (box.z - box.x) / RT + 1;
        const int tc = box.x + (int)(t % ntx) * RT, tr = box.y + (int)(t / ntx) * RT;
        const long long x0 = s.fx[id.x * 2], y0 = s.fx[id.x * 2 + 1], x1 = s.fx[id.y * 2], y1 = s.fx[id.y * 2 + 1];
        const long long x2 = s.fx[id.z * 2], y2 = s.fx[id.z * 2 + 1];
        const double z0 = s.vz[id.x], z1 = s.vz[id.y], z2 = s.vz[id.z];
        const double A = (double)edge(x0, y0, x1, y1, x2, y2);
        const bool tl12 = top_left(x1, y1, x2, y2), tl20 = top_left(x2, y2, x0, y0), tl01 = top_left(x0, y0, x1, y1);
        for (int k = lane; k < RT * RT; k += 32) {
            const int c = tc + (k % RT), r = tr + k / RT;
            if (c > box.z || r > box.w) continue;
            for (int q = 0; q < S; ++q) {
                const long long sx = 256ll * c + 128 + (S == 4 ? c_off4[q][0] : 0);
                const long long sy = 256ll * r + 128 + (S == 4 ? c_off4[q][1] : 0);
                const long long w0 = edge(x1, y1, x2, y2, sx, sy), w1 = edge(x2, y2, x0, y0, sx, sy), w2 = edge(x0, y0, x1, y1, sx, sy);
                if (!((w0 > 0 || (w0 == 0 && tl12)) && (w1 > 0 || (w1 == 0 && tl20)) && (w2 > 0 || (w2 == 0 && tl01)))) continue;
                float d = __double2float_rn(__ddiv_rn(da(da(dm((double)w0, z0), dm((double)w1, z1)), dm((double)w2, z2)), A));
                if (!(d >= -1.f && d <= 1.f)) continue;
                if (d == 0.f) d = 0.f;                                 // -0 and +0 are one depth
                unsigned b = __float_as_uint(d);
                b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
                const unsigned long long key = ((unsigned long long)b << 32) | (unsigned)f;
                unsigned long long* slot = s.keys + ((size_t)r * W + c) * S + q;
                if (key < *(volatile unsigned long long*)slot) atomicMin(slot, key);
            }
        }
    }
}

struct Shade {
    double base[3];
};

// pyrender mesh.frag, metallic 0, roughness 1 (see the header), one (pixel, face): returns the three bytes
__device__ void shade_face(const Scratch& s, int f, int c, int r, const Shade& sh, int out[3]) {
    const int4 id = s.fidx[f];
    const long long x0 = s.fx[id.x * 2], y0 = s.fx[id.x * 2 + 1], x1 = s.fx[id.y * 2], y1 = s.fx[id.y * 2 + 1];
    const long long x2 = s.fx[id.z * 2], y2 = s.fx[id.z * 2 + 1];
    const long long sx = 256ll * c + 128, sy = 256ll * r + 128;
    const double A = (double)edge(x0, y0, x1, y1, x2, y2);
    const double l0 = (double)edge(x1, y1, x2, y2, sx, sy) / A, l1 = (double)edge(x2, y2, x0, y0, sx, sy) / A;
    const double l2 = (double)edge(x0, y0, x1, y1, sx, sy) / A;
    double p[3], n[3];
    for (int j = 0; j < 3; ++j) {
        p[j] = da(da(dm(l0, s.pr[id.x * 3 + j]), dm(l1, s.pr[id.y * 3 + j])), dm(l2, s.pr[id.z * 3 + j]));
        n[j] = da(da(dm(l0, s.nrm[id.x * 3 + j]), dm(l1, s.nrm[id.y * 3 + j])), dm(l2, s.nrm[id.z * 3 + j]));
    }
    const double nl_ = sqrt(da(da(dm(n[0], n[0]), dm(n[1], n[1])), dm(n[2], n[2])));
    for (int j = 0; j < 3; ++j) n[j] = nl_ > 0.0 ? n[j] / nl_ : 0.0;
    const double pl = sqrt(da(da(dm(p[0], p[0]), dm(p[1], p[1])), dm(p[2], p[2])));
    double v[3] = {0.0, 0.0, 1.0};
    if (pl > 0.0)
        for (int j = 0; j < 3; ++j) v[j] = -p[j] / pl;
    const double nv = fmin(fmax(n[0] * v[0] + n[1] * v[1] + n[2] * v[2], 0.0), 1.0);
    const double L[3][3] = {{0.0, -1.0, 1.0}, {0.0, 1.0, 1.0}, {1.0, 1.0, 2.0}};
    double col[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < 3; ++k) {
        double l[3], h[3];
        for (int j = 0; j < 3; ++j) l[j] = L[k][j] - p[j];
        const double d2 = l[0] * l[0] + l[1] * l[1] + l[2] * l[2], d = sqrt(d2);
        for (int j = 0; j < 3; ++j) { l[j] /= d; h[j] = l[j] + v[j]; }
        const double hl = sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
        for (int j = 0; j < 3; ++j) h[j] = hl > 0.0 ? h[j] / hl : 0.0;
        const double nl = fmin(fmax(n[0] * l[0] + n[1] * l[1] + n[2] * l[2], 0.0), 1.0);
        const double vh = fmin(fmax(v[0] * h[0] + v[1] * h[1] + v[2] * h[2], 0.0), 1.0);
        const double om = 1.0 - vh, om2 = om * om;
        const double F = 0.04 + 0.96 * (om2 * om2 * om);
        const double G = (2.0 * nl / (nl + 1.0)) * (2.0 * nv / (nv + 1.0));
        const double spec = F * G * (1.0 / M_PI) / (4.0 * nl * nv + 0.001);
        for (int j = 0; j < 3; ++j) col[j] += nl * (1.0 / d2) * ((1.0 - F) * (0.96 * sh.base[j]) / M_PI + spec);
    }
    for (int j = 0; j < 3; ++j) {
        const double cj = fmin(fmax(pow(col[j] + 0.3 * sh.base[j], 1.0 / 2.2), 0.0), 1.0);
        out[j] = (int)floor(255.0 * cj + 0.5);
    }
}

__global__ void render_resolve_kernel(Scratch s, Shade sh, const unsigned char* __restrict__ img, int W, int H, int S,
                                      unsigned char* __restrict__ out, int* __restrict__ face_ids) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= W) return;
    const size_t pix = (size_t)r * W + c;
    int fid[4], byt[4][3], sum[3] = {0, 0, 0}, k = 0;
    for (int q = 0; q < S; ++q) {
        const unsigned long long key = s.keys[pix * S + q];
        fid[q] = key == EMPTY ? -1 : (int)(unsigned)(key & 0xffffffffu);
        if (face_ids) face_ids[pix * S + q] = fid[q];
        if (fid[q] < 0) continue;
        ++k;
        int same = -1;
        for (int p = 0; p < q; ++p)
            if (fid[p] == fid[q]) same = p;
        if (same >= 0)
            for (int j = 0; j < 3; ++j) byt[q][j] = byt[same][j];
        else
            shade_face(s, fid[q], c, r, sh, byt[q]);
        for (int j = 0; j < 3; ++j) sum[j] += byt[q][j];
    }
    for (int j = 0; j < 3; ++j) out[pix * 3 + j] = k ? (unsigned char)((sum[j] + S / 2) / S) : img[pix * 3 + j];
}

}  // namespace

long long render_scratch_bytes(int W, int H, int NV, int NF, int samples) {
    if (W < 1 || H < 1 || W > 8192 || H > 8192 || NV < 0 || NF < 0) return DBOA_ERR_SHAPE;
    if (samples != 1 && samples != 4) return DBOA_ERR_ARG;
    return (long long)carve(nullptr, nullptr, W, H, NV, NF, samples);
}

int render_overlay(const float* verts, const int* faces, const int* vf_offsets, const int* vf_faces, int NV, int NF, const float cam4[4],
                   const float rot3x3[9], const float color3[3], const unsigned char* img, int W, int H, int samples, void* scratch,
                   long long scratch_bytes, unsigned char* out, int* face_ids, cudaStream_t st) {
    const long long need = render_scratch_bytes(W, H, NV, NF, samples);
    if (need < 0) return (int)need;
    if (scratch_bytes < need) return DBOA_ERR_ARG;
    RenderCam c;
    c.sx = cam4[0]; c.sy = cam4[1]; c.tx = cam4[2]; c.ty = cam4[3];
    c.has_rot = rot3x3 != nullptr;
    for (int k = 0; k < 9; ++k) c.R[k] = rot3x3 ? (double)rot3x3[k] : (k % 4 == 0 ? 1.0 : 0.0);
    c.W = W; c.H = H; c.S = samples;
    Shade sh;
    for (int j = 0; j < 3; ++j) sh.base[j] = color3[j];
    Scratch s;
    carve(&s, (char*)scratch, W, H, NV, NF, samples);
    if (NV > 0) {
        render_vertex_kernel<<<ceil_div(NV, 128), 128, 0, st>>>(verts, NV, c, s);
        DBOA_TRY(check_launch());
        render_normal_kernel<<<ceil_div(NV, 128), 128, 0, st>>>(faces, NF, NV, vf_offsets, vf_faces, s);
        DBOA_TRY(check_launch());
    }
    if (NF > 0) {
        render_face_kernel<<<ceil_div(NF, 128), 128, 0, st>>>(faces, NF, NV, s, W, H);
        DBOA_TRY(check_launch());
    }
    render_scan_kernel<<<1, 1024, 0, st>>>(s.prefix, NF);
    DBOA_TRY(check_launch());
    if (cudaMemsetAsync(s.keys, 0xff, (size_t)W * H * samples * sizeof(unsigned long long), st) != cudaSuccess) return DBOA_ERR_CUDA;
    render_raster_kernel<<<num_sms() * 8, 256, 0, st>>>(NF, s, W, samples);
    DBOA_TRY(check_launch());
    render_resolve_kernel<<<dim3(ceil_div(W, 128), H), 128, 0, st>>>(s, sh, img, W, H, samples, out, face_ids);
    return check_launch();
}

}  // namespace dboa
