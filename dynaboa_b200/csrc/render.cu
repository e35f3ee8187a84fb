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
//
// Several meshes (render_overlay_groups): M <= 64 meshes of one topology, each over its own frame, in the same 6 kernels and
// 1 memset.  The per-mesh descriptors (RenderGroups) travel by value in a __grid_constant__ kernel parameter.  Vertex, normal
// and face kernels take the mesh from blockIdx.y, the scan runs one block per mesh, the raster walks the concatenated
// (mesh, face, tile) pairs of all meshes, the resolve gives each mesh its own run of row blocks.  Per (mesh, pixel, sample)
// the arithmetic is the one-mesh arithmetic, and no mesh reads another's scratch, so every mesh's out and face_ids are
// bit-identical to drawing it alone; render_overlay is the M = 1 call.
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

struct Shade {
    double base[3];
};

// one mesh of a grouped call: 256 bytes, so the table of 64 stays well inside the 32 KB kernel parameter space
struct RenderMesh {
    const float* verts;
    const unsigned char* img;
    unsigned char* out;
    int* face_ids;
    RenderCam c;
    Shade sh;
    Scratch s;
};

struct RenderGroups {
    RenderMesh m[64];
    int first_block[65];         // resolve: blocks [first_block[k], first_block[k + 1]) are mesh k's rows
    int n, NV, NF, S;
};

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Scratch layout: the vertex, face and prefix arrays of mesh 0, 1, ..., M - 1, then the depth keys of mesh 0, 1, ..., M - 1 as
// one region (one memset clears them all).  Every array starts on 256 bytes; M = 1 is the one-mesh layout.  Returns the
// byte size, and with s the arrays of each mesh and *keys_off the offset of the key region.
size_t carve(Scratch* s, char* base, const int* W, const int* H, int M, int NV, int NF, int S, size_t* keys_off = nullptr) {
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
    for (int k = 0; k < M; ++k) {
        char* pr = take((size_t)NV * 3 * sizeof(double));
        char* nrm = take((size_t)NV * 3 * sizeof(double));
        char* fx = take((size_t)NV * 2 * sizeof(long long));
        char* vz = take((size_t)NV * sizeof(double));
        char* vok = take((size_t)NV * sizeof(int));
        char* fidx = take((size_t)NF * sizeof(int4));
        char* fbox = take((size_t)NF * sizeof(int4));
        char* prefix = take(((size_t)NF + 1) * sizeof(long long));
        if (s) {
            s[k].pr = (double*)pr; s[k].nrm = (double*)nrm; s[k].fx = (long long*)fx; s[k].vz = (double*)vz; s[k].vok = (int*)vok;
            s[k].fidx = (int4*)fidx; s[k].fbox = (int4*)fbox; s[k].prefix = (long long*)prefix;
        }
    }
    if (keys_off) *keys_off = off;
    for (int k = 0; k < M; ++k) {
        char* keys = take((size_t)W[k] * H[k] * S * sizeof(unsigned long long));
        if (s) s[k].keys = (unsigned long long*)keys;
    }
    return off;
}

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dadd_rn(a, -b); }

__global__ void render_vertex_kernel(const __grid_constant__ RenderGroups g) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.NV) return;
    const RenderMesh& m = g.m[blockIdx.y];
    const float* __restrict__ verts = m.verts;
    const RenderCam& c = m.c;
    const Scratch& s = m.s;
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
__global__ void render_normal_kernel(const int* __restrict__ faces, const int* __restrict__ vf_off, const int* __restrict__ vf_faces,
                                     const __grid_constant__ RenderGroups g) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int NF = g.NF, NV = g.NV;
    if (i >= NV) return;
    const Scratch& s = g.m[blockIdx.y].s;
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
__global__ void render_face_kernel(const int* __restrict__ faces, const __grid_constant__ RenderGroups g) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    const int NF = g.NF, NV = g.NV;
    if (f >= NF) return;
    const RenderMesh& m = g.m[blockIdx.y];
    const Scratch& s = m.s;
    const int W = m.c.W, H = m.c.H;
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

// in-place inclusive scan of prefix[1..NF] by one block per mesh (the face count is small; this runs once per draw)
__global__ void __launch_bounds__(1024) render_scan_kernel(const __grid_constant__ RenderGroups g) {
    long long* __restrict__ prefix = g.m[blockIdx.x].s.prefix;
    const int NF = g.NF;
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

// grid-stride over the (mesh, face, tile) pairs of all meshes: mesh k owns the pairs [first[k], first[k + 1])
__global__ void __launch_bounds__(256) render_raster_kernel(const __grid_constant__ RenderGroups g) {
    __shared__ long long first[65];
    const int NF = g.NF, S = g.S, n = g.n;
    if (threadIdx.x < n) first[threadIdx.x + 1] = g.m[threadIdx.x].s.prefix[NF];
    __syncthreads();
    if (threadIdx.x == 0) {
        first[0] = 0;
        for (int k = 1; k <= n; ++k) first[k] += first[k - 1];
    }
    __syncthreads();
    const long long total = first[n];
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    int mk = 0;                                                        // a warp's pairs only grow: its mesh only advances
    for (long long gpair = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; gpair < total; gpair += nwarps) {
        while (first[mk + 1] <= gpair) ++mk;
        const Scratch s = g.m[mk].s;
        const int W = g.m[mk].c.W;
        const long long pair = gpair - first[mk];
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

// mesh k's (H, ceil(W / 128)) row blocks are the blocks [first_block[k], first_block[k + 1]) of a one-dimensional grid
__global__ void __launch_bounds__(128) render_resolve_kernel(const __grid_constant__ RenderGroups g) {
    int lo = 0, hi = g.n - 1;                                          // last mesh whose first block is <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (g.first_block[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const RenderMesh& m = g.m[lo];
    const Scratch& s = m.s;
    const int W = m.c.W, S = g.S;
    const int bx = (W + 127) / 128, b = (int)blockIdx.x - g.first_block[lo];
    const int c = (b % bx) * blockDim.x + threadIdx.x, r = b / bx;
    if (c >= W) return;
    const unsigned char* __restrict__ img = m.img;
    unsigned char* __restrict__ out = m.out;
    int* __restrict__ face_ids = m.face_ids;
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
            shade_face(s, fid[q], c, r, m.sh, byt[q]);
        for (int j = 0; j < 3; ++j) sum[j] += byt[q][j];
    }
    for (int j = 0; j < 3; ++j) out[pix * 3 + j] = k ? (unsigned char)((sum[j] + S / 2) / S) : img[pix * 3 + j];
}

}  // namespace

long long render_scratch_bytes_groups(const int* W, const int* H, int M, int NV, int NF, int samples) {
    if (!W || !H) return DBOA_ERR_ARG;
    if (M < 1 || M > 64 || NV < 0 || NF < 0) return DBOA_ERR_SHAPE;
    for (int k = 0; k < M; ++k)
        if (W[k] < 1 || H[k] < 1 || W[k] > 8192 || H[k] > 8192) return DBOA_ERR_SHAPE;
    if (samples != 1 && samples != 4) return DBOA_ERR_ARG;
    return (long long)carve(nullptr, nullptr, W, H, M, NV, NF, samples);
}

long long render_scratch_bytes(int W, int H, int NV, int NF, int samples) { return render_scratch_bytes_groups(&W, &H, 1, NV, NF, samples); }

int render_overlay_groups(const dboa_render_desc* meshes, int M, const int* faces, const int* vf_offsets, const int* vf_faces, int NV,
                          int NF, int samples, void* scratch, long long scratch_bytes, cudaStream_t st) {
    if (!meshes) return DBOA_ERR_ARG;
    if (M < 1 || M > 64) return DBOA_ERR_SHAPE;
    int W[64], H[64];
    for (int k = 0; k < M; ++k) { W[k] = meshes[k].W; H[k] = meshes[k].H; }
    const long long need = render_scratch_bytes_groups(W, H, M, NV, NF, samples);
    if (need < 0) return (int)need;
    for (int k = 0; k < M; ++k)
        if (!meshes[k].verts || !meshes[k].img || !meshes[k].out) return DBOA_ERR_ARG;
    if (scratch_bytes < need) return DBOA_ERR_ARG;
    RenderGroups g;
    g.n = M; g.NV = NV; g.NF = NF; g.S = samples;
    Scratch s[64];
    size_t keys_off = 0;
    carve(s, (char*)scratch, W, H, M, NV, NF, samples, &keys_off);
    long long blocks = 0;
    for (int k = 0; k < M; ++k) {
        const dboa_render_desc& d = meshes[k];
        RenderMesh& m = g.m[k];
        m.verts = d.verts; m.img = d.img; m.out = d.out; m.face_ids = d.face_ids;
        RenderCam& c = m.c;
        c.sx = d.cam4[0]; c.sy = d.cam4[1]; c.tx = d.cam4[2]; c.ty = d.cam4[3];
        c.has_rot = d.has_rot != 0;
        for (int j = 0; j < 9; ++j) c.R[j] = c.has_rot ? (double)d.rot3x3[j] : (j % 4 == 0 ? 1.0 : 0.0);
        c.W = W[k]; c.H = H[k]; c.S = samples;
        for (int j = 0; j < 3; ++j) m.sh.base[j] = d.color3[j];
        m.s = s[k];
        g.first_block[k] = (int)blocks;
        blocks += (long long)ceil_div(W[k], 128) * H[k];
    }
    g.first_block[M] = (int)blocks;                                     // <= 64 * 64 * 8192
    if (NV > 0) {
        render_vertex_kernel<<<dim3(ceil_div(NV, 128), M), 128, 0, st>>>(g);
        DBOA_TRY(check_launch());
        render_normal_kernel<<<dim3(ceil_div(NV, 128), M), 128, 0, st>>>(faces, vf_offsets, vf_faces, g);
        DBOA_TRY(check_launch());
    }
    if (NF > 0) {
        render_face_kernel<<<dim3(ceil_div(NF, 128), M), 128, 0, st>>>(faces, g);
        DBOA_TRY(check_launch());
    }
    render_scan_kernel<<<M, 1024, 0, st>>>(g);
    DBOA_TRY(check_launch());
    if (cudaMemsetAsync((char*)scratch + keys_off, 0xff, (size_t)need - keys_off, st) != cudaSuccess) return DBOA_ERR_CUDA;
    render_raster_kernel<<<num_sms() * 8, 256, 0, st>>>(g);
    DBOA_TRY(check_launch());
    render_resolve_kernel<<<(unsigned)blocks, 128, 0, st>>>(g);
    return check_launch();
}

int render_overlay(const float* verts, const int* faces, const int* vf_offsets, const int* vf_faces, int NV, int NF, const float cam4[4],
                   const float rot3x3[9], const float color3[3], const unsigned char* img, int W, int H, int samples, void* scratch,
                   long long scratch_bytes, unsigned char* out, int* face_ids, cudaStream_t st) {
    dboa_render_desc d;
    d.verts = verts; d.img = img; d.out = out; d.face_ids = face_ids;
    for (int j = 0; j < 4; ++j) d.cam4[j] = cam4[j];
    d.has_rot = rot3x3 != nullptr;
    for (int j = 0; j < 9; ++j) d.rot3x3[j] = rot3x3 ? rot3x3[j] : 0.f;
    for (int j = 0; j < 3; ++j) d.color3[j] = color3[j];
    d.W = W; d.H = H;
    return render_overlay_groups(&d, 1, faces, vf_offsets, vf_faces, NV, NF, samples, scratch, scratch_bytes, st);
}

}  // namespace dboa
