// Affinity pooling, the CSPN stereo network's convolutional spatial pyramid pooling: L levels of one feature map
// feat (B, C, H, W) pooled with learned affinities gate (B, L, H, W), forward and a deterministic backward, one launch each.
// Level l pools the windows of F.avg_pool2d(x, p) (stride p, no padding, floor mode) with p = p_l:
//
//   a(q) = |gate[b, l, q]|,  S = sum_{q in window} a(q),  w(q) = a(q) / S,  out_l[b, c, i, j] = sum_{q in window} w(q) feat[b, c, q]
//
// Operation order, every operation rounded on its own (no FMA contraction), every sum from its first term:
//   S, out      each window row summed in ascending x, then the row sums in ascending y
//   grad_feat   sum over the levels whose windows cover q, ascending l, of w_l(q) * grad_out_l[c, cell_l(q)]; +0.0 if none
//   grad_gate   t = sum_c grad_out_l[c] * (feat[c, q] - out_l[c]) in ascending c, then (t / S) * sgn(gate), sgn in {-1, 0, 1};
//               +0.0 outside level l's windows
// w is a / S in every result.  The bits depend on the arguments only: not on the tile, the stream, the batch split or the
// other levels of the call.
//
// Kernels.  The forward runs every level in one launch: a CTA owns one level's cell row i, a run of J cells of it and a
// chunk of ch channels, with J and ch chosen per level so that a thread does about the same work at every level (a
// p = 64 window is not the tail).  A thread owns one window row of one cell and sums it for the chunk's channels with w
// computed once per pixel; the window's row sums then meet in shared memory and one thread per (cell, channel) adds them.
// The backward owns 4 x 32 pixel tiles: it recomputes S of every window that meets the tile, in the forward's order, and
// then a thread owns one pixel and both of its gradients, walking the channels.  Both gradients are gathers: no atomics,
// no workspace, no memset; every output element is written once.
#include <algorithm>

#include "common.cuh"

namespace cspn {
namespace {

constexpr int kFwdThreads = 128;
constexpr int kWork = 128;            // target window-row terms per forward thread: ch * p
constexpr int kMaxCh = 16;
constexpr int kTileY = 4, kTileX = 32, kBwdThreads = kTileY * kTileX;
constexpr int kRowBuf = 1024;         // backward: row sums of one chunk of window rows

struct Level {
    int p, Hl, Wl;
    int J, ch, yc;                    // forward: cells per CTA, channels per CTA, window rows per chunk
    long long out_off;                // first element of the level in the packed output
    long long block0;                 // first forward CTA of the level
};

struct Levels {
    Level lv[kAffinityPoolMaxLevels];
    int L;
};

// The cells of a level (n of them along the axis, width p) that meet [t0, t0 + tn)
__device__ __forceinline__ int tile_cells(int t0, int tn, int p, int n) {
    const int end = min(t0 + tn, n * p);
    return t0 < end ? (end - 1) / p - t0 / p + 1 : 0;
}

__device__ __forceinline__ float sgn_of(float g) { return (float)(g > 0.f) - (float)(g < 0.f); }

// S of the ny x nx windows of one level starting at cell (i0, j0): each window row summed in ascending x, then the rows in
// ascending y.  Rows are summed in chunks of yc rows (ncell * yc <= rows_cap slots of `rows`); thread k < ncell keeps
// window k's running sum and stores it to s[k].  All threads of the CTA call it.
__device__ __forceinline__ void window_sums(const float* __restrict__ g, int W, int p, int i0, int j0, int ny, int nx, int yc, float* rows,
                            float* s) {
    const int ncell = ny * nx;
    float run = 0.f;
    for (int y0 = 0; y0 < p; y0 += yc) {
        const int nr = min(yc, p - y0);
        __syncthreads();                                  // the last chunk's rows are consumed
        for (int t = threadIdx.x; t < ncell * nr; t += blockDim.x) {
            const int k = t % ncell, yy = t / ncell;
            const float* row = g + (size_t)((i0 + k / nx) * p + y0 + yy) * W + (size_t)(j0 + k % nx) * p;
            float r = fabsf(__ldg(row));
            for (int x = 1; x < p; ++x) r = __fadd_rn(r, fabsf(__ldg(row + x)));
            rows[yy * ncell + k] = r;
        }
        __syncthreads();
        if (threadIdx.x < ncell)
            for (int yy = 0; yy < nr; ++yy) {
                const float r = rows[yy * ncell + threadIdx.x];
                run = (y0 == 0 && yy == 0) ? r : __fadd_rn(run, r);
            }
    }
    if (threadIdx.x < ncell) s[threadIdx.x] = run;
    __syncthreads();
}

// ---- forward: grid (sum over levels of B * channel chunks * Hl * cell runs) ---------------------------------------------------
template <int CH>
__device__ __forceinline__ void pool_level(const float* __restrict__ feat, const float* __restrict__ g, float* __restrict__ out, int C, int H,
                           int W, const Level& v, int b, int c0, int nc, int i, int j0, int nj, float* sm) {
    const int p = v.p, yc = v.yc;
    float* sS = sm;                                       // [J]
    float* rows = sS + v.J;                               // [J * yc]: gate row sums, then channel row sums [CH][nj][yc + 1]
    window_sums(g, W, p, i, j0, 1, nj, yc, rows, sS);
    const size_t plane = (size_t)H * W;
    const int pitch = yc + 1;
    const int own_c = threadIdx.x / max(nj, 1), own_j = threadIdx.x % max(nj, 1);    // the (cell, channel) this thread adds
    float tot = 0.f;
    for (int y0 = 0; y0 < p; y0 += yc) {
        const int nr = min(yc, p - y0);
        if (y0 > 0) __syncthreads();                      // the last chunk's row sums are consumed
        if (threadIdx.x < nj * nr) {
            const int jl = threadIdx.x % nj, y = i * p + y0 + threadIdx.x / nj, x0 = (j0 + jl) * p;
            const float S = sS[jl];
            const float* grow = g + (size_t)y * W + x0;
            const float* frow = feat + (size_t)c0 * plane + (size_t)y * W + x0;
            float acc[CH];
            {
                const float w = __fdiv_rn(fabsf(__ldg(grow)), S);
#pragma unroll
                for (int k = 0; k < CH; ++k)
                    if (k < nc) acc[k] = __fmul_rn(w, __ldg(frow + k * plane));
            }
            for (int x = 1; x < p; ++x) {
                const float w = __fdiv_rn(fabsf(__ldg(grow + x)), S);
#pragma unroll
                for (int k = 0; k < CH; ++k)
                    if (k < nc) acc[k] = __fadd_rn(acc[k], __fmul_rn(w, __ldg(frow + k * plane + x)));
            }
            float* dst = rows + jl * pitch + threadIdx.x / nj;
#pragma unroll
            for (int k = 0; k < CH; ++k)
                if (k < nc) dst[k * nj * pitch] = acc[k];
        }
        __syncthreads();
        if (threadIdx.x < nj * nc)
            for (int yy = 0; yy < nr; ++yy) {
                const float r = rows[(own_c * nj + own_j) * pitch + yy];
                tot = (y0 == 0 && yy == 0) ? r : __fadd_rn(tot, r);
            }
    }
    if (threadIdx.x < nj * nc) out[(((size_t)b * C + c0 + own_c) * v.Hl + i) * v.Wl + j0 + own_j] = tot;
}

__global__ void __launch_bounds__(kFwdThreads)
affinity_pool_fwd_kernel(const float* __restrict__ feat, const float* __restrict__ gate, float* __restrict__ out, int B, int C,
                         int H, int W, const __grid_constant__ Levels P) {
    extern __shared__ float smem[];
    int l = 0;
    while (l + 1 < P.L && P.lv[l + 1].block0 <= (long long)blockIdx.x) ++l;
    const Level& v = P.lv[l];
    long long r = (long long)blockIdx.x - v.block0;
    const int runs = (v.Wl + v.J - 1) / v.J, chunks = (C + v.ch - 1) / v.ch;
    const int jr = (int)(r % runs);
    r /= runs;
    const int i = (int)(r % v.Hl);
    r /= v.Hl;
    const int cc = (int)(r % chunks), b = (int)(r / chunks);
    const int j0 = jr * v.J, nj = min(v.J, v.Wl - j0), c0 = cc * v.ch, nc = min(v.ch, C - c0);
    const float* f = feat + (size_t)b * C * H * W;
    const float* g = gate + ((size_t)b * P.L + l) * H * W;
    float* o = out + v.out_off;
    switch (v.ch) {
        case 1: pool_level<1>(f, g, o, C, H, W, v, b, c0, nc, i, j0, nj, smem); break;
        case 2: pool_level<2>(f, g, o, C, H, W, v, b, c0, nc, i, j0, nj, smem); break;
        case 4: pool_level<4>(f, g, o, C, H, W, v, b, c0, nc, i, j0, nj, smem); break;
        case 8: pool_level<8>(f, g, o, C, H, W, v, b, c0, nc, i, j0, nj, smem); break;
        default: pool_level<kMaxCh>(f, g, o, C, H, W, v, b, c0, nc, i, j0, nj, smem); break;
    }
}

// ---- backward: grid (B * tiles), a 4 x 32 pixel tile per CTA, a pixel per thread -------------------------------------------
__global__ void __launch_bounds__(kBwdThreads, 4)
affinity_pool_bwd_kernel(const float* __restrict__ feat, const float* __restrict__ gate, const float* __restrict__ out,
                         const float* __restrict__ gout, float* __restrict__ gfeat, float* __restrict__ ggate, int B, int C,
                         int H, int W, const __grid_constant__ Levels P) {
    __shared__ float sS[kAffinityPoolMaxLevels][kBwdThreads];
    __shared__ float rows[kRowBuf];
    const int tiles_x = (W + kTileX - 1) / kTileX, tiles = tiles_x * ((H + kTileY - 1) / kTileY);
    const int b = (int)(blockIdx.x / tiles), tile = (int)(blockIdx.x % tiles);
    const int y0 = tile / tiles_x * kTileY, x0 = tile % tiles_x * kTileX;
    const int y = y0 + threadIdx.x / kTileX, x = x0 + threadIdx.x % kTileX;
    const int L = P.L;
    const size_t plane = (size_t)H * W;
    // S of every window that meets the tile, per level, in the forward's order, to sS[l][(i - i0) * nx + j - j0]
#pragma unroll 1
    for (int l = 0; l < L; ++l) {
        const Level& v = P.lv[l];
        const int i0 = y0 / v.p, j0 = x0 / v.p, ny = tile_cells(y0, kTileY, v.p, v.Hl), nx = tile_cells(x0, kTileX, v.p, v.Wl);
        if (ny * nx > 0)                                  // uniform over the CTA
            window_sums(gate + ((size_t)b * L + l) * plane, W, v.p, i0, j0, ny, nx, max(1, min(v.p, kRowBuf / (ny * nx))),
                        rows, sS[l]);
    }
    if (y >= H || x >= W) return;
    int sidx[kAffinityPoolMaxLevels];                     // the pixel's window in sS[l], or -1 outside level l's windows
#pragma unroll
    for (int l = 0; l < kAffinityPoolMaxLevels; ++l) {
        sidx[l] = -1;
        if (l >= L) continue;
        const Level& v = P.lv[l];
        if (y < v.Hl * v.p && x < v.Wl * v.p) sidx[l] = (y / v.p - y0 / v.p) * tile_cells(x0, kTileX, v.p, v.Wl) + x / v.p - x0 / v.p;
    }
    const size_t px = (size_t)y * W + x;
    float w[kAffinityPoolMaxLevels], t[kAffinityPoolMaxLevels];
    size_t cell[kAffinityPoolMaxLevels];                  // the pixel's cell in level l at channel 0 (sidx[l] >= 0)
#pragma unroll
    for (int l = 0; l < kAffinityPoolMaxLevels; ++l) {
        if (sidx[l] < 0) continue;
        const Level& v = P.lv[l];
        w[l] = __fdiv_rn(fabsf(__ldg(gate + ((size_t)b * L + l) * plane + px)), sS[l][sidx[l]]);
        cell[l] = v.out_off + ((size_t)b * C * v.Hl + y / v.p) * v.Wl + x / v.p;
    }
    for (int c = 0; c < C; ++c) {
        const size_t fo = ((size_t)b * C + c) * plane + px;
        const float f = __ldg(feat + fo);
        float gf = 0.f;
        bool first = true;
#pragma unroll
        for (int l = 0; l < kAffinityPoolMaxLevels; ++l) {
            if (sidx[l] < 0) continue;
            const Level& v = P.lv[l];
            const size_t o = cell[l] + (size_t)c * v.Hl * v.Wl;
            const float go = __ldg(gout + o);
            const float term = __fmul_rn(w[l], go);
            gf = first ? term : __fadd_rn(gf, term);
            first = false;
            const float pr = __fmul_rn(go, __fsub_rn(f, __ldg(out + o)));
            t[l] = c == 0 ? pr : __fadd_rn(t[l], pr);
        }
        gfeat[fo] = gf;
    }
#pragma unroll
    for (int l = 0; l < kAffinityPoolMaxLevels; ++l) {
        if (l >= L) continue;
        const size_t go = ((size_t)b * L + l) * plane + px;
        ggate[go] = sidx[l] < 0 ? 0.f : __fmul_rn(__fdiv_rn(t[l], sS[l][sidx[l]]), sgn_of(__ldg(gate + go)));
    }
}

long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

// The per-level forward plan: J cells of p rows each fill at most a CTA of threads, ch = the power of two nearest below
// kWork / p (1 to 32) with J * ch <= threads (one adding thread per (cell, channel)); rows in chunks of yc <= threads.
Levels plan_levels(int B, int C, int H, int W, int L, const int* ks, size_t* smem, long long* blocks) {
    Levels P{};
    P.L = L;
    long long off = 0, blk = 0;
    size_t sm = 0;
    for (int l = 0; l < L; ++l) {
        Level& v = P.lv[l];
        v.p = ks[l];
        v.Hl = H / v.p;
        v.Wl = W / v.p;
        v.J = std::max(1, std::min(kFwdThreads / v.p, v.Wl));
        v.yc = std::min(v.p, kFwdThreads);
        int ch = 1;
        while (ch < kMaxCh && 2 * ch * v.p <= kWork) ch *= 2;
        while (ch > 1 && v.J * ch > kFwdThreads) ch /= 2;
        v.ch = ch;
        v.out_off = off;
        v.block0 = blk;
        off += (long long)B * C * v.Hl * v.Wl;
        blk += (long long)B * ceil_div(C, ch) * v.Hl * ceil_div(v.Wl, v.J);
        sm = std::max(sm, (size_t)(v.J + std::max(v.J * v.yc, ch * v.J * (v.yc + 1))) * sizeof(float));
    }
    *smem = sm;
    *blocks = blk;
    return P;
}

}  // namespace

int affinity_pool_launchable(int B, int C, int H, int W, int L, const int* kernel_sizes, const char** why) {
    if ((long long)H * W >= (1ll << 31)) { *why = "a (B, channel) slice has >= 2^31 elements"; return 0; }
    size_t smem;
    long long blocks;
    plan_levels(B, C, H, W, L, kernel_sizes, &smem, &blocks);
    if (blocks >= (1ll << 31)) { *why = "the forward grid has >= 2^31 blocks"; return 0; }
    if ((long long)B * ceil_div(H, kTileY) * ceil_div(W, kTileX) >= (1ll << 31)) {
        *why = "the backward grid has >= 2^31 blocks";
        return 0;
    }
    return 1;
}

int affinity_pool_forward(const float* feat, const float* gate, float* out, int B, int C, int H, int W, int L,
                          const int* kernel_sizes, cudaStream_t st, int* launches) {
    size_t smem;
    long long blocks;
    const Levels P = plan_levels(B, C, H, W, L, kernel_sizes, &smem, &blocks);
    affinity_pool_fwd_kernel<<<(unsigned)blocks, kFwdThreads, smem, st>>>(feat, gate, out, B, C, H, W, P);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

int affinity_pool_backward(const float* feat, const float* gate, const float* out, const float* grad_out, float* grad_feat,
                           float* grad_gate, int B, int C, int H, int W, int L, const int* kernel_sizes, cudaStream_t st,
                           int* launches) {
    size_t smem;
    long long blocks;
    const Levels P = plan_levels(B, C, H, W, L, kernel_sizes, &smem, &blocks);
    const long long tiles = (long long)B * ceil_div(H, kTileY) * ceil_div(W, kTileX);
    affinity_pool_bwd_kernel<<<(unsigned)tiles, kBwdThreads, 0, st>>>(feat, gate, out, grad_out, grad_feat, grad_gate, B, C, H,
                                                                       W, P);
    CSPN_CUDA_TRY(cudaGetLastError());
    *launches = 1;
    return CSPN_OK;
}

}  // namespace cspn
