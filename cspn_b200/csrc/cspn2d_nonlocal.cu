// Non-local 2D propagation, NLSPN's (Park et al., ECCV 2020): every one of a pixel's T = K*K - 1 neighbours sits at a
// learned, fractional offset from its grid position and is read by bilinear sampling (DESIGN.md section 4.21).  feat
// (B, C, H, W) is h_0; offset (B, 2T, H, W) holds (dy, dx) of tap k in channels 2k, 2k + 1; affinity (B, T, H, W) holds
// a_k, used as given and shared by the C channels; sparse (B, C, H, W) is optional.  Tap k runs over (i, j) in [0, K)^2 in
// raster order without the centre, base offset (i - R, j - R), R = (K - 1) / 2.  With S(h, y, x) torchvision's
// bilinear_interpolate (0 when y <= -1, y >= H, x <= -1 or x >= W; NaN for a NaN position; a corner outside the image
// contributes nothing, one inside contributes weight * value even when the weight is 0):
//
//   a_c = 1 - sum_k a_k                     (sum from a_0, k ascending)
//   h_{t+1}(p) = a_c S(h~_t, p) + sum_k a_k S(h~_t, p + base_k + delta_k(p))
//              = a_c * S_c + (a_0 S_0 + a_1 S_1 + ...)        (the tap sum from its first term, then the centre added)
//   h~_t = (1 - m) h_t + m sparse,  m = 1[sparse > 0]        (only with a sparse; h_N, the output, is not replaced)
//
// S = ((w_tl v_tl + w_tr v_tr) + w_bl v_bl) + w_br v_br with w_tl = hy hx, w_tr = hy lx, w_bl = ly hx, w_br = ly lx, ly =
// y - floor(y), hy = 1 - ly (x alike).  Every product and sum is rounded on its own: no FMA contraction.
//
// Backward, with lambda_N = grad_out and lambda~_t the adjoint of h~_t:
//   lambda~_t(q) = a_c(q) lambda_{t+1}(q) + sum over the samples (p, k) that have q as a corner of (a_k(p) w) lambda_{t+1}(p)
//   lambda_t = (1 - m) lambda~_t,  grad_feat = lambda_0,  grad_sparse = sum_t m lambda~_t (t ascending)
//   grad_affinity_k(p) = G_k - G_c,  G_k = sum_t sum_c lambda_{t+1} S_k(h~_t),  G_c the same sum of S_c
//   grad_offset_{2k}(p) = sum_t sum_c (a_k cw_y(h~_t)) lambda_{t+1},  cw_y = lx (v_br - v_tr) + hx (v_bl - v_tl)
//   grad_offset_{2k+1}(p) = sum_t sum_c (a_k cw_x(h~_t)) lambda_{t+1},  cw_x = ly (v_br - v_bl) + hy (v_tr - v_tl)
// sums over t then c ascending, from their first term.  As in torchvision's deform_conv2d backward, a corner whose weight
// is exactly 0 (the lower or right one at an integer coordinate) takes no part in the adjoint, and cw has no window test:
// it is the right-sided derivative, built from the corners at floor and floor + 1 that lie in the image.
//
// The adjoint is a gather: every sample (p, k) whose position lies in (-1, H) x (-1, W) is listed once under its top-left
// corner, in an (H + 1) x (W + 1) bucket grid per image.  A stable radix sort by bucket of the list in (b, k, p) order
// keeps each bucket's entries in ascending (k, p), so pixel q sums its buckets q, q - (0, 1), q - (1, 0), q - (1, 1) in
// that order, each in ascending (k, p): the bits depend on the arguments only, never on timing.
//
// Kernels (sm_90a):
//   forward   one launch per step, a thread per pixel and up to kCh channels, h~ ping-ponging in the workspace;
//   backward  1. N - 1 forward steps store h~_1 .. h~_{N-1} (the first also h~_0 in replacement mode), only when the
//                affinity or offset gradient is requested;
//             2. the bucket keys and the a_c planes; the radix sort (CUB); the bucket starts (a binary search per
//                bucket); the entries' corner weights a_k w;
//             3. N adjoint gathers, the last one also writing grad_feat and grad_sparse;
//             4. one finalize kernel, a thread per (b, k, p), for grad_affinity and grad_offset (t, then c ascending).
// No floating-point atomics: only the radix sort (CUB) uses integer atomics and memsets, for its own counters.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace cspn {
namespace {

constexpr int kThreads = 128;
constexpr int kCh = 4;                       // channels per thread
constexpr unsigned kNoXHigh = 1u << 30;      // entry flags: the right corners have weight 0 (lx == 0)
constexpr unsigned kNoYHigh = 1u << 29;      //              the lower corners have weight 0 (ly == 0)
constexpr unsigned kPixMask = (1u << 29) - 1;

// One bilinear sample's geometry: the four corners tl, tr, bl, br, which of them lie in the image, their weights, and
// whether S is 0 (outside the window), NaN (a NaN coordinate) or the weighted sum
struct Samp {
    int o[4];
    unsigned in;
    float ly, lx, hy, hx;
    int kind;                                // 0: S = 0, 1: S = NaN, 2: bilinear
};

__device__ __forceinline__ Samp make_samp(float y, float x, int H, int W) {
    Samp s;
    s.kind = (y <= -1.f || y >= (float)H || x <= -1.f || x >= (float)W) ? 0 : ((y == y && x == x) ? 2 : 1);
    const float y0 = floorf(y), x0 = floorf(x);          // float floor: no huge or non-finite value becomes an int
    s.ly = __fsub_rn(y, y0);
    s.lx = __fsub_rn(x, x0);
    s.hy = __fsub_rn(1.f, s.ly);
    s.hx = __fsub_rn(1.f, s.lx);
    const float y1 = __fadd_rn(y0, 1.f), x1 = __fadd_rn(x0, 1.f);
    const bool vy0 = y0 >= 0.f && y0 < (float)H, vy1 = y1 >= 0.f && y1 < (float)H;
    const bool vx0 = x0 >= 0.f && x0 < (float)W, vx1 = x1 >= 0.f && x1 < (float)W;
    const int iy0 = vy0 ? (int)y0 : 0, iy1 = vy1 ? (int)y1 : 0, ix0 = vx0 ? (int)x0 : 0, ix1 = vx1 ? (int)x1 : 0;
    s.o[0] = iy0 * W + ix0;
    s.o[1] = iy0 * W + ix1;
    s.o[2] = iy1 * W + ix0;
    s.o[3] = iy1 * W + ix1;
    s.in = (unsigned)(vy0 && vx0) | (unsigned)(vy0 && vx1) << 1 | (unsigned)(vy1 && vx0) << 2 | (unsigned)(vy1 && vx1) << 3;
    return s;
}

__device__ __forceinline__ float replaced(float h, float sp) {
    const float m = sp > 0.f ? 1.f : 0.f;
    return __fadd_rn(__fmul_rn(__fsub_rn(1.f, m), h), __fmul_rn(m, sp));
}

// The four corner values of plane h (0 outside the image); kRep: h~ = the replacement of h by the sparse plane sp
template <bool kRep>
__device__ __forceinline__ void corners(const Samp& s, const float* __restrict__ h, const float* __restrict__ sp, float v[4]) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        v[r] = 0.f;
        if (s.in >> r & 1u) {
            v[r] = __ldg(h + s.o[r]);
            if (kRep) v[r] = replaced(v[r], __ldg(sp + s.o[r]));
        }
    }
}

__device__ __forceinline__ float bilinear(const Samp& s, const float v[4]) {
    if (s.kind == 0) return 0.f;
    if (s.kind == 1) return __int_as_float(0x7fc00000);
    float acc = __fmul_rn(__fmul_rn(s.hy, s.hx), v[0]);
    acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(s.hy, s.lx), v[1]));
    acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(s.ly, s.hx), v[2]));
    return __fadd_rn(acc, __fmul_rn(__fmul_rn(s.ly, s.lx), v[3]));
}

// Tap k of a K x K kernel: its base offset (i - R, j - R), (i, j) raster order without the centre
template <int K>
__device__ __forceinline__ void tap_base(int k, int& di, int& dj) {
    constexpr int R = (K - 1) / 2, T = K * K - 1;
    const int idx = k < T / 2 ? k : k + 1;
    di = idx / K - R;
    dj = idx % K - R;
}

// ---- forward step: grid (pixel blocks, B * channel chunks) ------------------------------------------------------------------
// hin = h~_t (or feat when kRepRead: h~_0 formed from feat and sp on the fly); hout = h~_{t+1} (replaced when kRepWrite)
// or h_N; h0out, when not null, receives h~_0 at the thread's own pixel (the backward's recomputation, replacement mode)
template <int K, bool kRepRead, bool kRepWrite>
__global__ void __launch_bounds__(kThreads)
nl_step_kernel(const float* __restrict__ hin, const float* __restrict__ sp, const float* __restrict__ off,
               const float* __restrict__ aff, float* __restrict__ hout, float* __restrict__ h0out, int C, int H, int W, int chunks) {
    constexpr int T = K * K - 1;
    const int HW = H * W;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= HW) return;
    const int cc = blockIdx.y % chunks, b = blockIdx.y / chunks;
    const int py = p / W, px = p - py * W;
    const int c0 = cc * kCh, nc = min(kCh, C - c0);
    const size_t plane = (size_t)HW;
    const float* hb = hin + ((size_t)b * C + c0) * plane;
    const float* sb = kRepRead ? sp + ((size_t)b * C + c0) * plane : nullptr;
    const float* ob = off + (size_t)b * 2 * T * plane + p;
    const float* ab = aff + (size_t)b * T * plane + p;
    float acc[kCh], sum = 0.f;
#pragma unroll 1
    for (int k = 0; k < T; ++k) {
        const float a = __ldg(ab + k * plane);
        int di, dj;
        tap_base<K>(k, di, dj);
        const Samp s = make_samp(__fadd_rn((float)(py + di), __ldg(ob + 2 * k * plane)),
                                 __fadd_rn((float)(px + dj), __ldg(ob + (2 * k + 1) * plane)), H, W);
        sum = k == 0 ? a : __fadd_rn(sum, a);
#pragma unroll
        for (int j = 0; j < kCh; ++j) {
            if (j >= nc) break;
            float v[4];
            corners<kRepRead>(s, hb + j * plane, kRepRead ? sb + j * plane : nullptr, v);
            const float term = __fmul_rn(a, bilinear(s, v));
            acc[j] = k == 0 ? term : __fadd_rn(acc[j], term);
        }
    }
    const float ac = __fsub_rn(1.f, sum);
    const Samp s = make_samp((float)py, (float)px, H, W);
    float* ho = hout + ((size_t)b * C + c0) * plane + p;
    const float* sw = kRepWrite ? sp + ((size_t)b * C + c0) * plane + p : nullptr;
#pragma unroll
    for (int j = 0; j < kCh; ++j) {
        if (j >= nc) break;
        float v[4];
        corners<kRepRead>(s, hb + j * plane, kRepRead ? sb + j * plane : nullptr, v);
        float h = __fadd_rn(__fmul_rn(ac, bilinear(s, v)), acc[j]);
        if (kRepWrite) h = replaced(h, __ldg(sw + j * plane));
        ho[j * plane] = h;
        if (h0out) h0out[((size_t)b * C + c0 + j) * plane + p] = v[0];   // v[0] is h~_0 at p itself
    }
}

// ---- backward 2a: the bucket keys of every sample, grid (pixel blocks, T, B), and the a_c planes (threads of tap 0) --------
template <int K>
__global__ void __launch_bounds__(kThreads)
nl_keys_kernel(const float* __restrict__ off, const float* __restrict__ aff, unsigned* __restrict__ keys, int* __restrict__ vals,
               float* __restrict__ acp, int H, int W, unsigned NB, unsigned sentinel) {
    constexpr int T = K * K - 1;
    const int HW = H * W;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= HW) return;
    const int k = blockIdx.y, b = blockIdx.z;
    const int py = p / W, px = p - py * W;
    const size_t plane = (size_t)HW;
    const float* ob = off + (size_t)b * 2 * T * plane + p;
    int di, dj;
    tap_base<K>(k, di, dj);
    const float y = __fadd_rn((float)(py + di), __ldg(ob + 2 * k * plane));
    const float x = __fadd_rn((float)(px + dj), __ldg(ob + (2 * k + 1) * plane));
    unsigned key = sentinel;
    if (y > -1.f && y < (float)H && x > -1.f && x < (float)W)     // false for NaN: such a sample has no corner
        key = (unsigned)b * NB + (unsigned)((int)floorf(y) + 1) * (unsigned)(W + 1) + (unsigned)((int)floorf(x) + 1);
    const size_t e = ((size_t)b * T + k) * plane + p;
    keys[e] = key;
    vals[e] = k * HW + p;
    if (k == 0) {
        const float* ab = aff + (size_t)b * T * plane + p;
        float sum = __ldg(ab);
#pragma unroll 1
        for (int j = 1; j < T; ++j) sum = __fadd_rn(sum, __ldg(ab + j * plane));
        acp[(size_t)b * plane + p] = __fsub_rn(1.f, sum);
    }
}

// ---- backward 2b: start[j] = the first sorted position whose key is >= j, j = 0 .. B * NB -----------------------------------
__global__ void __launch_bounds__(kThreads)
nl_starts_kernel(const unsigned* __restrict__ keys, long long n, long long nb, long long* __restrict__ start) {
    for (long long j = (long long)blockIdx.x * kThreads + threadIdx.x; j <= nb; j += (long long)gridDim.x * kThreads) {
        long long lo = 0, hi = n;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (__ldg(keys + mid) < (unsigned long long)j) lo = mid + 1;
            else hi = mid;
        }
        start[j] = lo;
    }
}

// ---- backward 2c: per sorted entry, its pixel (with the zero-weight flags) and a_k w for the four corner roles -------------
template <int K>
__global__ void __launch_bounds__(kThreads)
nl_entries_kernel(const unsigned* __restrict__ keys, const int* __restrict__ vals, const float* __restrict__ off,
                  const float* __restrict__ aff, unsigned* __restrict__ ent_p, float* __restrict__ ent_w, long long n, int H, int W,
                  unsigned NB, unsigned sentinel) {
    constexpr int T = K * K - 1;
    const int HW = H * W;
    const size_t plane = (size_t)HW;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const unsigned key = __ldg(keys + i);
        if (key >= sentinel) continue;                  // a sample with no corner in the image: never read by the adjoint
        const int b = (int)(key / NB);
        const int v = __ldg(vals + i), k = v / HW, p = v - k * HW;
        const int py = p / W, px = p - py * W;
        int di, dj;
        tap_base<K>(k, di, dj);
        const float* ob = off + (size_t)b * 2 * T * plane + p;
        const Samp s = make_samp(__fadd_rn((float)(py + di), __ldg(ob + 2 * k * plane)),
                                 __fadd_rn((float)(px + dj), __ldg(ob + (2 * k + 1) * plane)), H, W);
        const float a = __ldg(aff + ((size_t)b * T + k) * plane + p);
        ent_p[i] = (unsigned)p | (s.lx == 0.f ? kNoXHigh : 0u) | (s.ly == 0.f ? kNoYHigh : 0u);
        ent_w[i] = __fmul_rn(a, __fmul_rn(s.hy, s.hx));
        ent_w[n + i] = __fmul_rn(a, __fmul_rn(s.hy, s.lx));
        ent_w[2 * n + i] = __fmul_rn(a, __fmul_rn(s.ly, s.hx));
        ent_w[3 * n + i] = __fmul_rn(a, __fmul_rn(s.ly, s.lx));
    }
}

// ---- backward 3: one adjoint step, grid (pixel blocks, B * channel chunks) ----------------------------------------------------
// lam_in = lambda_{t+1}; writes lambda~_t to lt (when not null), lambda_t = (1 - m) lambda~_t to lam_out (when not null);
// the last step (t = 0) writes grad_feat = lambda_0 and grad_sparse = sum_t m lambda~_t over lambda~_1.. in slots, t ascending
__global__ void __launch_bounds__(kThreads)
nl_adjoint_kernel(const float* __restrict__ lam_in, const float* __restrict__ acp, const float* __restrict__ sp,
                  const long long* __restrict__ start, const unsigned* __restrict__ ent_p, const float* __restrict__ ent_w, long long n,
                  float* __restrict__ lt, float* __restrict__ lam_out, float* __restrict__ gfeat, float* __restrict__ gsp,
                  const float* __restrict__ slots, int n_slots, size_t slot, int C, int H, int W, int chunks, unsigned NB) {
    const int HW = H * W;
    const int q = blockIdx.x * kThreads + threadIdx.x;
    if (q >= HW) return;
    const int cc = blockIdx.y % chunks, b = blockIdx.y / chunks;
    const int qy = q / W, qx = q - qy * W;
    const int c0 = cc * kCh, nc = min(kCh, C - c0);
    const size_t plane = (size_t)HW, cbase = ((size_t)b * C + c0) * plane;
    const float* li = lam_in + cbase;
    const float ac = __ldg(acp + (size_t)b * plane + q);
    float acc[kCh];
#pragma unroll
    for (int j = 0; j < kCh; ++j)
        if (j < nc) acc[j] = __fmul_rn(ac, __ldg(li + j * plane + q));
    const size_t bb = (size_t)b * NB;
#pragma unroll
    for (int r = 0; r < 4; ++r) {                                 // q as the tl, tr, bl, br corner of the bucket's samples
        const int by = qy + 1 - (r >> 1), bx = qx + 1 - (r & 1);
        const size_t bk = bb + (size_t)by * (W + 1) + bx;
        const long long e0 = __ldg(start + bk), e1 = __ldg(start + bk + 1);
        const unsigned skip = ((r & 1) ? kNoXHigh : 0u) | ((r >> 1) ? kNoYHigh : 0u);
        const float* wr = ent_w + (size_t)r * n;
#pragma unroll 1
        for (long long i = e0; i < e1; ++i) {
            const unsigned pe = __ldg(ent_p + i);
            if (pe & skip) continue;
            const int p = (int)(pe & kPixMask);
            const float w = __ldg(wr + i);
#pragma unroll
            for (int j = 0; j < kCh; ++j)
                if (j < nc) acc[j] = __fadd_rn(acc[j], __fmul_rn(w, __ldg(li + j * plane + p)));
        }
    }
#pragma unroll
    for (int j = 0; j < kCh; ++j) {
        if (j >= nc) break;
        const size_t e = cbase + j * plane + q;
        const float m = sp ? (__ldg(sp + e) > 0.f ? 1.f : 0.f) : 0.f;
        const float lam = sp ? __fmul_rn(__fsub_rn(1.f, m), acc[j]) : acc[j];
        if (lt) lt[e] = acc[j];
        if (lam_out) lam_out[e] = lam;
        if (gfeat) gfeat[e] = lam;
        if (gsp) {
            float g = __fmul_rn(m, acc[j]);
#pragma unroll 1
            for (int t = 1; t < n_slots; ++t) g = __fadd_rn(g, __fmul_rn(m, __ldg(slots + (size_t)t * slot + e)));
            gsp[e] = g;
        }
    }
}

// ---- backward 4: grad_affinity and grad_offset, grid (pixel blocks, T, B) -------------------------------------------------------
// hs: slot t = h~_t (slot 0 = feat without replacement); ls: slot t = lambda~_t for t >= 1; lambda_{t+1} = (1 - m) lambda~_{t+1}
// is formed again here with the adjoint's bits, lambda_N = grad_out
template <int K>
__global__ void __launch_bounds__(kThreads)
nl_finalize_kernel(const float* __restrict__ feat, const float* __restrict__ hs, const float* __restrict__ ls,
                   const float* __restrict__ gout, const float* __restrict__ sp, const float* __restrict__ off,
                   const float* __restrict__ aff, float* __restrict__ gaff, float* __restrict__ goff, int N, int B, int C, int H, int W) {
    constexpr int T = K * K - 1;
    const int HW = H * W;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= HW) return;
    const int k = blockIdx.y, b = blockIdx.z;
    const int py = p / W, px = p - py * W;
    const size_t plane = (size_t)HW, slot = (size_t)B * C * plane;
    const float* ob = off + (size_t)b * 2 * T * plane + p;
    int di, dj;
    tap_base<K>(k, di, dj);
    const Samp s = make_samp(__fadd_rn((float)(py + di), __ldg(ob + 2 * k * plane)),
                             __fadd_rn((float)(px + dj), __ldg(ob + (2 * k + 1) * plane)), H, W);
    const Samp sc = make_samp((float)py, (float)px, H, W);
    const float a = __ldg(aff + ((size_t)b * T + k) * plane + p);
    float gk = 0.f, gc = 0.f, gy = 0.f, gx = 0.f;
    bool first = true;
#pragma unroll 1
    for (int t = 0; t < N; ++t) {
        const float* h = (t == 0 && !sp) ? feat : hs + (size_t)t * slot;
#pragma unroll 1
        for (int c = 0; c < C; ++c) {
            const size_t pl = ((size_t)b * C + c) * plane;
            float lam;
            if (t + 1 == N) lam = __ldg(gout + pl + p);
            else {
                lam = __ldg(ls + (size_t)(t + 1) * slot + pl + p);
                if (sp) lam = __fmul_rn(__fsub_rn(1.f, __ldg(sp + pl + p) > 0.f ? 1.f : 0.f), lam);
            }
            float v[4], vc[4];
            corners<false>(s, h + pl, nullptr, v);
            corners<false>(sc, h + pl, nullptr, vc);
            const float tk = __fmul_rn(lam, bilinear(s, v)), tc = __fmul_rn(lam, bilinear(sc, vc));
            gk = first ? tk : __fadd_rn(gk, tk);
            gc = first ? tc : __fadd_rn(gc, tc);
            if (goff) {
                const float cy = __fadd_rn(__fmul_rn(s.lx, __fsub_rn(v[3], v[1])), __fmul_rn(s.hx, __fsub_rn(v[2], v[0])));
                const float cx = __fadd_rn(__fmul_rn(s.ly, __fsub_rn(v[3], v[2])), __fmul_rn(s.hy, __fsub_rn(v[1], v[0])));
                const float ty = __fmul_rn(__fmul_rn(a, cy), lam), tx = __fmul_rn(__fmul_rn(a, cx), lam);
                gy = first ? ty : __fadd_rn(gy, ty);
                gx = first ? tx : __fadd_rn(gx, tx);
            }
            first = false;
        }
    }
    if (gaff) gaff[((size_t)b * T + k) * plane + p] = __fsub_rn(gk, gc);
    if (goff) {
        goff[((size_t)b * 2 * T + 2 * k) * plane + p] = gy;
        goff[((size_t)b * 2 * T + 2 * k + 1) * plane + p] = gx;
    }
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }
size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// The backward workspace's regions, in bytes from its start
struct BwdLayout {
    size_t hs, ls, lp, ac, keys, vals, entw, start, temp, total, temp_bytes;
};

int key_bits(unsigned long long sentinel) {
    int bits = 1;
    while (bits < 32 && (sentinel >> bits) != 0) ++bits;
    return bits;
}

bool sort_temp_bytes(long long n, int bits, size_t* bytes) {
    cub::DoubleBuffer<unsigned> k(nullptr, nullptr);
    cub::DoubleBuffer<int> v(nullptr, nullptr);
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, k, v, n, 0, bits) == cudaSuccess;
}

bool bwd_layout(int B, int C, int H, int W, int K, int N, BwdLayout* L) {
    const long long T = (long long)K * K - 1, hw = (long long)H * W, P = (long long)B * C * hw, n = (long long)B * hw * T;
    const unsigned long long nb = (unsigned long long)B * (H + 1) * (W + 1);
    size_t o = 0;
    L->hs = o;    o = align256(o + (size_t)N * P * 4);
    L->ls = o;    o = align256(o + (size_t)N * P * 4);
    L->lp = o;    o = align256(o + (size_t)2 * P * 4);
    L->ac = o;    o = align256(o + (size_t)B * hw * 4);
    L->keys = o;  o = align256(o + (size_t)2 * n * 4);
    L->vals = o;  o = align256(o + (size_t)2 * n * 4);
    L->entw = o;  o = align256(o + (size_t)4 * n * 4);
    L->start = o; o = align256(o + (size_t)(nb + 1) * 8);
    if (!sort_temp_bytes(n, key_bits(nb), &L->temp_bytes)) return false;
    L->temp = o;  o = align256(o + L->temp_bytes);
    L->total = o + 256;                      // the regions are laid out from the first 256-byte boundary of the workspace
    return true;
}

template <int K>
int forward_k(const float* feat, const float* offset, const float* affinity, const float* sparse, float* out, int B, int C, int H,
              int W, int N, void* ws, cudaStream_t st, int* launches) {
    const int HW = H * W, chunks = (int)ceil_div(C, kCh);
    const dim3 grid((unsigned)ceil_div(HW, kThreads), (unsigned)(B * chunks));
    float* buf[2] = {static_cast<float*>(ws), static_cast<float*>(ws) + (size_t)B * C * HW};
    const float* hin = feat;
    for (int t = 0; t < N; ++t) {
        const bool last = t + 1 == N;
        float* hout = last ? out : buf[t & 1];
        if (sparse && t == 0)
            last ? nl_step_kernel<K, true, false><<<grid, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, nullptr, C, H, W, chunks)
                 : nl_step_kernel<K, true, true><<<grid, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, nullptr, C, H, W, chunks);
        else if (sparse && !last)
            nl_step_kernel<K, false, true><<<grid, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, nullptr, C, H, W, chunks);
        else
            nl_step_kernel<K, false, false><<<grid, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, nullptr, C, H, W, chunks);
        CSPN_CUDA_TRY(cudaGetLastError());
        hin = hout;
    }
    *launches = N;
    return CSPN_OK;
}

template <int K>
int backward_k(const float* feat, const float* offset, const float* affinity, const float* sparse, const float* grad_out,
               float* grad_feat, float* grad_offset, float* grad_affinity, float* grad_sparse, int B, int C, int H, int W, int N,
               void* ws, cudaStream_t st, int* launches) {
    constexpr int T = K * K - 1;
    BwdLayout L;
    if (!bwd_layout(B, C, H, W, K, N, &L)) { set_error("cannot size the radix sort's scratch"); return CSPN_ERR_CUDA; }
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);   // the ABI takes 4-byte alignment
    const int HW = H * W, chunks = (int)ceil_div(C, kCh);
    const size_t P = (size_t)B * C * HW;
    const long long n = (long long)B * HW * T;
    const unsigned NB = (unsigned)((H + 1) * (W + 1));
    const unsigned long long nb = (unsigned long long)B * NB;
    const bool need_hist = grad_affinity || grad_offset;          // the finalize: h~_t and lambda_{t+1} for every t
    const bool need_slots = need_hist || grad_sparse;
    float* hs = reinterpret_cast<float*>(base + L.hs);
    float* ls = reinterpret_cast<float*>(base + L.ls);
    float* lp = reinterpret_cast<float*>(base + L.lp);
    float* acp = reinterpret_cast<float*>(base + L.ac);
    unsigned* keys = reinterpret_cast<unsigned*>(base + L.keys);
    int* vals = reinterpret_cast<int*>(base + L.vals);
    float* entw = reinterpret_cast<float*>(base + L.entw);
    long long* start = reinterpret_cast<long long*>(base + L.start);
    int nl = 0;
    const dim3 pix((unsigned)ceil_div(HW, kThreads), (unsigned)(B * chunks));
    const dim3 taps((unsigned)ceil_div(HW, kThreads), (unsigned)T, (unsigned)B);
    // 1. h~_1 .. h~_{N-1} (and h~_0 with a sparse), only for the finalize
    if (need_hist) {
        for (int t = 0; t + 1 < N; ++t) {
            const float* hin = t == 0 ? feat : hs + (size_t)t * P;
            float* hout = hs + (size_t)(t + 1) * P;
            if (sparse && t == 0)
                nl_step_kernel<K, true, true><<<pix, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, hs, C, H, W, chunks);
            else if (sparse)
                nl_step_kernel<K, false, true><<<pix, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, nullptr, C, H, W, chunks);
            else
                nl_step_kernel<K, false, false><<<pix, kThreads, 0, st>>>(hin, sparse, offset, affinity, hout, nullptr, C, H, W, chunks);
            CSPN_CUDA_TRY(cudaGetLastError());
            ++nl;
        }
        if (sparse && N == 1) {        // h~_0 alone: a step whose output is discarded into the first lambda plane
            nl_step_kernel<K, true, false><<<pix, kThreads, 0, st>>>(feat, sparse, offset, affinity, lp, hs, C, H, W, chunks);
            CSPN_CUDA_TRY(cudaGetLastError());
            ++nl;
        }
    }
    // 2. the transposed index: keys, sort, bucket starts, entries
    const int t_end = (grad_feat || grad_sparse) ? 0 : 1;        // the last adjoint step to run
    if (N - 1 >= t_end) {
        const unsigned sentinel = (unsigned)nb;
        nl_keys_kernel<K><<<taps, kThreads, 0, st>>>(offset, affinity, keys, vals, acp, H, W, NB, sentinel);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
        cub::DoubleBuffer<unsigned> kb(keys, keys + n);
        cub::DoubleBuffer<int> vb(vals, vals + n);
        size_t temp = L.temp_bytes;
        CSPN_CUDA_TRY(cub::DeviceRadixSort::SortPairs(base + L.temp, temp, kb, vb, n, 0, key_bits(nb), st));
        nl += 1;
        const unsigned* sk = kb.Current();
        const int* sv = vb.Current();
        unsigned* ent_p = reinterpret_cast<unsigned*>(vb.Alternate());
        const unsigned blocks = (unsigned)min((long long)ceil_div((long long)nb + 1, kThreads), 1ll << 20);
        nl_starts_kernel<<<blocks, kThreads, 0, st>>>(sk, n, (long long)nb, start);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
        nl_entries_kernel<K><<<(unsigned)min(ceil_div(n, kThreads), 1ll << 20), kThreads, 0, st>>>(
            sk, sv, offset, affinity, ent_p, entw, n, H, W, NB, sentinel);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
        // 3. the adjoint, t = N-1 down to t_end
        for (int t = N - 1; t >= t_end; --t) {
            const float* lam_in = t + 1 == N ? grad_out : lp + (size_t)((t + 1) & 1) * P;
            float* lt = (need_slots && t >= 1) ? ls + (size_t)t * P : nullptr;
            float* lam_out = t >= 1 ? lp + (size_t)(t & 1) * P : nullptr;
            nl_adjoint_kernel<<<pix, kThreads, 0, st>>>(lam_in, acp, sparse, start, ent_p, entw, n, lt, lam_out,
                                                        t == 0 ? grad_feat : nullptr, t == 0 ? grad_sparse : nullptr, ls, N,
                                                        P, C, H, W, chunks, NB);
            CSPN_CUDA_TRY(cudaGetLastError());
            ++nl;
        }
    }
    // 4. grad_affinity and grad_offset
    if (need_hist) {
        nl_finalize_kernel<K><<<taps, kThreads, 0, st>>>(feat, hs, ls, grad_out, sparse, offset, affinity, grad_affinity, grad_offset,
                                                         N, B, C, H, W);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
    }
    *launches = nl;
    return CSPN_OK;
}

}  // namespace

int nonlocal2d_launchable(int B, int C, int H, int W, int K, const char** why) {
    const long long T = (long long)K * K - 1, hw = (long long)H * W;
    if (hw * T >= (1ll << 31)) { *why = "H*W*T >= 2^31 (the transposed index holds int32 entries)"; return 0; }
    if ((long long)B * ceil_div(C, kCh) > 65535) { *why = "B*ceil(C/4) exceeds gridDim.y (65535)"; return 0; }
    if ((unsigned long long)B * (H + 1) * (W + 1) >= (1ull << 32) - 1) { *why = "B*(H+1)*(W+1) >= 2^32 - 1 buckets"; return 0; }
    return 1;
}

size_t nonlocal2d_workspace_bytes(int B, int C, int H, int W, int N) {
    const int bufs = N < 2 ? 0 : (N == 2 ? 1 : 2);
    return (size_t)bufs * B * C * H * W * sizeof(float);
}

size_t nonlocal2d_bwd_workspace_bytes(int B, int C, int H, int W, int K, int N) {
    if (N == 0) return 0;
    BwdLayout L;
    return bwd_layout(B, C, H, W, K, N, &L) ? L.total : 0;
}

int nonlocal2d_forward(const float* feat, const float* offset, const float* affinity, const float* sparse, float* out, int B, int C,
                       int H, int W, int K, int N, void* ws, cudaStream_t st, int* launches) {
    if (N == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(out, feat, (size_t)B * C * H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
        *launches = 0;
        return CSPN_OK;
    }
    switch (K) {
        case 3: return forward_k<3>(feat, offset, affinity, sparse, out, B, C, H, W, N, ws, st, launches);
        case 5: return forward_k<5>(feat, offset, affinity, sparse, out, B, C, H, W, N, ws, st, launches);
        default: return forward_k<7>(feat, offset, affinity, sparse, out, B, C, H, W, N, ws, st, launches);
    }
}

int nonlocal2d_backward(const float* feat, const float* offset, const float* affinity, const float* sparse, const float* grad_out,
                        float* grad_feat, float* grad_offset, float* grad_affinity, float* grad_sparse, int B, int C, int H, int W,
                        int K, int N, void* ws, cudaStream_t st, int* launches) {
    if (N == 0) {      // h_0 = feat: the identity, and nothing reaches the offsets, the affinities or the samples
        const size_t hw = (size_t)H * W, T = (size_t)K * K - 1;
        if (grad_feat) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_feat, grad_out, (size_t)B * C * hw * 4, cudaMemcpyDeviceToDevice, st));
        if (grad_offset) CSPN_CUDA_TRY(cudaMemsetAsync(grad_offset, 0, (size_t)B * 2 * T * hw * 4, st));
        if (grad_affinity) CSPN_CUDA_TRY(cudaMemsetAsync(grad_affinity, 0, (size_t)B * T * hw * 4, st));
        if (grad_sparse) CSPN_CUDA_TRY(cudaMemsetAsync(grad_sparse, 0, (size_t)B * C * hw * 4, st));
        *launches = 0;
        return CSPN_OK;
    }
    switch (K) {
        case 3: return backward_k<3>(feat, offset, affinity, sparse, grad_out, grad_feat, grad_offset, grad_affinity, grad_sparse, B, C, H,
                                     W, N, ws, st, launches);
        case 5: return backward_k<5>(feat, offset, affinity, sparse, grad_out, grad_feat, grad_offset, grad_affinity, grad_sparse, B, C, H,
                                     W, N, ws, st, launches);
        default: return backward_k<7>(feat, offset, affinity, sparse, grad_out, grad_feat, grad_offset, grad_affinity, grad_sparse, B, C,
                                      H, W, N, ws, st, launches);
    }
}

}  // namespace cspn
