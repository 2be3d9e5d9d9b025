// 3D CSPN with a K x K x K affinity kernel, K = 2R+1 = 5 (K^3-1 = 124 neighbours), forward and backward, and the 3x3x3
// backward (R = 1).  The 3x3x3 forward keeps its own kernels (cspn3d.cu); the C ABI delegates it to them.
//
// Arithmetic: cspn3d.cu with K^3-1 taps (at K = 3 its taps in its order: Taps3<1> is off3_*).  Tap k enumerates (f, t, l)
// over [0,K)^3 in raster order without the centre (R, R, R) and reads the source at (dz, dy, dx) = (R-f, R-t, R-l)
// (oracle/cspn_numpy_3d_k.py::offsets_3d):
//   gathered (mode 0 signed, 1 abs): a_k(p) = ghat_k(p + off_k) (0 outside),  w_k = a_k / sum_j |a_j|,  kappa = 1 - sum_k w_k,
//                                    d_{t+1} = kappa d0 + sum_k w_k d_t(p + off_k);
//   'paddle' (mode 2):               w_k(p) = |g_k(p)| / sum_j |g_j(p)| at the voxel's own location, no centre term.
//
// Why not cspn3d.cu's design at K = 5: its step keeps 9 rows x 6 floats of the current volume and 26 weights in registers.
// 124 weights per voxel and 25 rows x 8 floats do not fit, so
//   'paddle'  each step reads the 124 raw guidance planes at the voxel's own location (streamed in chunks of one z-slab of
//             the window, 25 loads in flight per thread), sums |g| and divides once per voxel.  No prep, no weight planes;
//   gathered  one prep launch per volume group writes w_k and kappa (K^3 = 125 planes per volume); each step streams them.
// Both steps stage the CTA's tile of d_t plus an R-voxel halo in z, y and x in shared memory (zeros outside the volume).
// W % 4 == 0 with 16-byte aligned pointers: 4 consecutive voxels per thread, every plane read as LDG.128; otherwise one
// voxel per thread.  Volume groups: group3d with K^3 planes per volume.
// Backward, in the staged form of cspn2d_wide.cu, one volume at a time: prep (for 'paddle' too), N-1 forward steps that keep
// d_1..d_{N-1}, N adjoint steps lambda_t(q) = sum_k w_k(q - off_k) lambda_{t+1}(q - off_k) that keep every lambda_t
// (lambda_{t+1} tile + halo in shared memory), K gather launches -- one per z-slab of the window, 25 register accumulators
// Gw_k(p) = sum_c sum_t lambda_{t+1}(p) d_t(p + off_k) each, written over the then dead weight planes -- and one finalize
// with the chain rule (fin3k_kernel).
//
// Caller-supplied gates (fluid.layers.affinity_propagate itself, DESIGN.md section 4.11), K in {3, 5}:
//   d_{t+1}(p) = sum_k g_k(p) d_t(p + off_k)   with the gates used as given (no |.|, no division, no centre term).
// The step kernels' RAW mode reads the caller's gates [vol][NT][V] as the weight planes: no prep, no cold-sum branch.  The
// backward runs the staged form above on the gates themselves: the adjoint reads the volume's gates, the last adjoint writes
// lambda_0 straight into grad_feat, and the K gather launches write Gw_k straight into grad_gates (no prep, no finalize).
//
// Fused gather (cspn3d_{,k_,gates_}fwd_gather_f32, DESIGN.md section 4.6): the FAN flag of the two step kernels, as in
// cspn3d.cu: only the last step of a launch group stores to the other GPUs' gather buffers.
#include <cstdlib>

#include "common.cuh"

namespace cspn {

namespace {

template <int R>
struct Taps3 {
    static constexpr int K = 2 * R + 1;
    static constexpr int NT = K * K * K - 1;   // neighbours = guidance channels
    static constexpr int NP = K * K * K;       // planes per volume in the workspace: w_0..w_{NT-1}, kappa
    __host__ __device__ static constexpr int idx(int k) { return k >= NT / 2 ? k + 1 : k; }
    __host__ __device__ static constexpr int dz(int k) { return R - idx(k) / (K * K); }
    __host__ __device__ static constexpr int dy(int k) { return R - (idx(k) / K) % K; }
    __host__ __device__ static constexpr int dx(int k) { return R - idx(k) % K; }
    // the tap of window position (f, t, l) != (R, R, R)
    __host__ __device__ static constexpr int tap(int f, int t, int l) {
        return (f * K + t) * K + l - ((f * K + t) * K + l > NT / 2 ? 1 : 0);
    }
};

__device__ __forceinline__ bool inside3(int z, int y, int x, int D, int H, int W) {
    return z >= 0 && z < D && y >= 0 && y < H && x >= 0 && x < W;
}

// streaming load of a plane that is read once per step (guidance / weight planes)
__device__ __forceinline__ float4 ld_stream4(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// ---- prep: w_k and kappa of every voxel.  grid z = volume of the group * D + z ------------------------------------
// At R = 2 the guidance is read twice (sum, then quotients) instead of holding 124 values per thread; the 26 of R = 1 stay
// in registers and are read once.
template <int R>
__device__ __forceinline__ float prep_tap(const float* __restrict__ g, int k, int z, int y, int x, int D, int H, int W,
                                          size_t V, size_t p, int mode) {
    using T = Taps3<R>;
    if (mode == 2) return fabsf(__ldg(g + k * V + p));
    const int zz = z + T::dz(k), yy = y + T::dy(k), xx = x + T::dx(k);
    if (!inside3(zz, yy, xx, D, H, W)) return 0.f;
    const float v = __ldg(g + k * V + ((size_t)zz * H + yy) * W + xx);
    return mode == 1 ? fabsf(v) : v;
}

template <int R>
__global__ void __launch_bounds__(256)
prep3k_kernel(const float* __restrict__ g, float* __restrict__ wk, int D, int H, int W, int mode) {
    using T = Taps3<R>;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z % D, vol = blockIdx.z / D;
    if (x >= W || y >= H) return;
    const size_t V = (size_t)D * H * W, p = ((size_t)z * H + y) * W + x;
    g += (size_t)vol * T::NT * V;
    wk += (size_t)vol * T::NP * V;
    constexpr int U = R == 1 ? T::NT : 4;   // unroll: R = 1 fully, so that a[] is registers
    float a[R == 1 ? T::NT : 1];
    float S = 0.f;
#pragma unroll U
    for (int k = 0; k < T::NT; ++k) {
        const float v = prep_tap<R>(g, k, z, y, x, D, H, W, V, p, mode);
        if constexpr (R == 1) a[k] = v;
        S += fabsf(v);
    }
    float s = 0.f;
#pragma unroll U
    for (int k = 0; k < T::NT; ++k) {
        float v;
        if constexpr (R == 1) v = a[k];
        else v = prep_tap<R>(g, k, z, y, x, D, H, W, V, p, mode);
        const float w = __fdiv_rn(v, S);   // IEEE: 0/0 NaN, x/inf 0
        s += w;
        wk[k * V + p] = w;
    }
    wk[T::NT * V + p] = mode == 2 ? 0.f : 1.f - s;
}

// ---- step, 4 voxels of a row per thread (W % 4 == 0, 16-byte aligned pointers) ----------------------------------
// CTA tile 64 x 16 voxels of one z-plane, 16 x 16 threads.  The shared tile holds planes z-R .. z+R, rows y0-R .. y0+15+R
// and columns x0-4 .. x0+67 as float4 (the halo rounded up to 4 columns: a thread's window row is three aligned LDS.128).
// PADDLE: w = raw guidance [vol][NT][V], out = sum_k |g_k| d_t(p+off_k) / sum_k |g_k|.  RAW: w = the caller's gates
// [vol][NT][V], out = sum_k g_k d_t(p+off_k).  Otherwise w = weight planes [vol][NP][V], out = kappa d0 + sum_k w_k
// d_t(p+off_k), or without the kappa term when d0 is null ('paddle' planes).  FAN: the result also goes to fan's
// destinations (the last step of a fused gather); fan is not read otherwise.
constexpr int kVecTW = 64, kVecTH = 16;

template <int R, bool PADDLE, bool RAW = false, bool FAN = false>
__global__ void __launch_bounds__(256)
step3k_vec_kernel(const float* __restrict__ w, const float* __restrict__ d0, const float* __restrict__ cur,
                  float* __restrict__ dst, int C, int D, int H, int W, const Fan fan) {
    using T = Taps3<R>;
    constexpr int SZ = 2 * R + 1, SH = kVecTH + 2 * R, SQ = kVecTW / 4 + 2;
    __shared__ float4 tile[SZ][SH][SQ];
    const int x0 = blockIdx.x * kVecTW, y0 = blockIdx.y * kVecTH;
    const int z = blockIdx.z % D, bc = blockIdx.z / D;   // bc = volume * C + channel
    const size_t HW = (size_t)H * W, V = (size_t)D * HW;
    const float* c = cur + (size_t)bc * V;
    for (int i = threadIdx.y * 16 + threadIdx.x; i < SZ * SH * SQ; i += 256) {
        const int q = i % SQ, r = (i / SQ) % SH, f = i / (SQ * SH);
        const int gz = z - R + f, gy = y0 - R + r, gx = x0 - 4 + 4 * q;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (inside3(gz, gy, gx, D, H, W)) v = __ldg(reinterpret_cast<const float4*>(c + (size_t)gz * HW + (size_t)gy * W + gx));
        tile[f][r][q] = v;
    }
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int x = x0 + 4 * tx, y = y0 + ty;
    if (x >= W || y >= H) return;
    const size_t p = (size_t)z * HW + (size_t)y * W + x;
    const float* wp = w + (size_t)(bc / C) * (PADDLE || RAW ? T::NT : T::NP) * V + p;
    float acc[4] = {0.f, 0.f, 0.f, 0.f}, S[4] = {0.f, 0.f, 0.f, 0.f};
    if (!PADDLE && !RAW && d0) {
        const float4 kap = ld_stream4(wp + T::NT * V);
        const float4 dd = __ldg(reinterpret_cast<const float4*>(d0 + (size_t)bc * V + p));
        acc[0] = kap.x * dd.x; acc[1] = kap.y * dd.y; acc[2] = kap.z * dd.z; acc[3] = kap.w * dd.w;
    }
#pragma unroll 1
    for (int f = 0; f < T::K; ++f) {   // one z-slab of the window per iteration: its 25 (24) plane loads issued back to back
        float4 wl[T::K * T::K];
#pragma unroll
        for (int j = 0; j < T::K * T::K; ++j)
            wl[j] = (j == T::K * T::K / 2 && f == R) ? make_float4(0.f, 0.f, 0.f, 0.f)
                                                      : ld_stream4(wp + (size_t)T::tap(f, j / T::K, j % T::K) * V);
#pragma unroll
        for (int t = 0; t < T::K; ++t) {
            const float4* tr = tile[2 * R - f][ty + 2 * R - t];   // source plane z + (R-f), row y + (R-t)
            const float4 A = tr[tx], B = tr[tx + 1], Cq = tr[tx + 2];
            const float row[12] = {A.x, A.y, A.z, A.w, B.x, B.y, B.z, B.w, Cq.x, Cq.y, Cq.z, Cq.w};   // columns x-4 .. x+7
#pragma unroll
            for (int l = 0; l < T::K; ++l) {
                if (t == R && l == R && f == R) continue;
                const int dx = R - l;
                float4 wv = wl[t * T::K + l];
                if (PADDLE) {
                    wv = make_float4(fabsf(wv.x), fabsf(wv.y), fabsf(wv.z), fabsf(wv.w));
                    S[0] += wv.x; S[1] += wv.y; S[2] += wv.z; S[3] += wv.w;
                }
                acc[0] = fmaf(wv.x, row[4 + dx], acc[0]);
                acc[1] = fmaf(wv.y, row[5 + dx], acc[1]);
                acc[2] = fmaf(wv.z, row[6 + dx], acc[2]);
                acc[3] = fmaf(wv.w, row[7 + dx], acc[3]);
            }
        }
    }
    if (PADDLE) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (cold_paddle(S[j], acc[j])) {   // cold: form the quotients one by one, as the weight planes hold them
                float a = 0.f;
                // by 4, as ptxas unrolls it at R = 2: unrolled 26 times at R = 1, the division calls cost a spill
#pragma unroll 4
                for (int k = 0; k < T::NT; ++k) {
                    const float* tr = reinterpret_cast<const float*>(tile[R + T::dz(k)][ty + R + T::dy(k)] + tx);
                    a = fmaf(__fdiv_rn(fabsf(__ldg(wp + k * V + j)), S[j]), tr[4 + j + T::dx(k)], a);
                }
                acc[j] = a;
            } else {
                acc[j] = __fdiv_rn(acc[j], S[j]);
            }
        }
    }
    const size_t o = (size_t)bc * V + p;
    const float4 v = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(dst + o) = v;
    if constexpr (FAN) fan_store(fan, o, v);
}

// ---- step / adjoint, one voxel per thread (any W, any alignment).  Tile 32 x 8 voxels of one z-plane + R halo ----
constexpr int kSclTW = 32, kSclTH = 8;

template <int R>
__device__ __forceinline__ void load_tile3_scalar(float (*tile)[kSclTH + 2 * R][kSclTW + 2 * R], const float* __restrict__ src,
                                                  int x0, int y0, int z, int D, int H, int W) {
    constexpr int SZ = 2 * R + 1, SH = kSclTH + 2 * R, SW = kSclTW + 2 * R;
    for (int i = threadIdx.y * kSclTW + threadIdx.x; i < SZ * SH * SW; i += kSclTW * kSclTH) {
        const int q = i % SW, r = (i / SW) % SH, f = i / (SW * SH);
        const int gz = z - R + f, gy = y0 - R + r, gx = x0 - R + q;
        tile[f][r][q] = inside3(gz, gy, gx, D, H, W) ? __ldg(src + ((size_t)gz * H + gy) * W + gx) : 0.f;
    }
}

template <int R, bool PADDLE, bool RAW = false, bool FAN = false>
__global__ void __launch_bounds__(256)
step3k_scalar_kernel(const float* __restrict__ w, const float* __restrict__ d0, const float* __restrict__ cur,
                     float* __restrict__ dst, int C, int D, int H, int W, const Fan fan) {
    using T = Taps3<R>;
    __shared__ float tile[2 * R + 1][kSclTH + 2 * R][kSclTW + 2 * R];
    const int x0 = blockIdx.x * kSclTW, y0 = blockIdx.y * kSclTH;
    const int z = blockIdx.z % D, bc = blockIdx.z / D;
    const size_t V = (size_t)D * H * W;
    load_tile3_scalar<R>(tile, cur + (size_t)bc * V, x0, y0, z, D, H, W);
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    if (x >= W || y >= H) return;
    const size_t p = ((size_t)z * H + y) * W + x;
    const float* wp = w + (size_t)(bc / C) * (PADDLE || RAW ? T::NT : T::NP) * V + p;
    float acc = (!PADDLE && !RAW && d0) ? __ldg(wp + T::NT * V) * __ldg(d0 + (size_t)bc * V + p) : 0.f, S = 0.f;
#pragma unroll 1
    for (int f = 0; f < T::K; ++f) {
#pragma unroll
        for (int t = 0; t < T::K; ++t) {
#pragma unroll
            for (int l = 0; l < T::K; ++l) {
                if (t == R && l == R && f == R) continue;
                float wv = __ldg(wp + (size_t)T::tap(f, t, l) * V);
                if (PADDLE) { wv = fabsf(wv); S += wv; }
                acc = fmaf(wv, tile[2 * R - f][ty + 2 * R - t][tx + 2 * R - l], acc);
            }
        }
    }
    if (PADDLE) {
        if (cold_paddle(S, acc)) {
            acc = 0.f;
            for (int k = 0; k < T::NT; ++k)
                acc = fmaf(__fdiv_rn(fabsf(__ldg(wp + k * V)), S), tile[R + T::dz(k)][ty + R + T::dy(k)][tx + R + T::dx(k)], acc);
        } else {
            acc = __fdiv_rn(acc, S);
        }
    }
    const size_t o = (size_t)bc * V + p;
    dst[o] = acc;
    if constexpr (FAN) fan_store(fan, o, acc);
}

// lambda_t(q) = sum_k w_k(q - off_k) lambda_{t+1}(q - off_k): the transposed stencil over source voxels inside the volume.
// One volume: grid z = channel * D + z.
template <int R>
__global__ void __launch_bounds__(256)
adj3k_kernel(const float* __restrict__ wk, const float* __restrict__ lam_in, float* __restrict__ lam_out, int D, int H, int W) {
    using T = Taps3<R>;
    __shared__ float tile[2 * R + 1][kSclTH + 2 * R][kSclTW + 2 * R];
    const int x0 = blockIdx.x * kSclTW, y0 = blockIdx.y * kSclTH;
    const int z = blockIdx.z % D, c = blockIdx.z / D;
    const size_t V = (size_t)D * H * W;
    load_tile3_scalar<R>(tile, lam_in + (size_t)c * V, x0, y0, z, D, H, W);
    __syncthreads();
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    if (x >= W || y >= H) return;
    float acc = 0.f;
#pragma unroll 1
    for (int f = 0; f < T::K; ++f) {
        const int zs = z - (R - f);
        if (zs < 0 || zs >= D) continue;
#pragma unroll
        for (int t = 0; t < T::K; ++t) {
#pragma unroll
            for (int l = 0; l < T::K; ++l) {
                if (t == R && l == R && f == R) continue;
                const int ys = y - (R - t), xs = x - (R - l);
                if (ys >= 0 && ys < H && xs >= 0 && xs < W)
                    acc = fmaf(__ldg(wk + (size_t)T::tap(f, t, l) * V + ((size_t)zs * H + ys) * W + xs), tile[f][ty + t][tx + l], acc);
            }
        }
    }
    lam_out[(size_t)c * V + ((size_t)z * H + y) * W + x] = acc;
}

// Gw_k(p) = sum_c sum_t lambda_{t+1}(p) d_t(p + off_k) for the taps of z-slab f of the window (dz = R - f), with the d_t
// plane z + dz staged tile by tile; written to plane k of gw.  steps[t] = d_{t+1}, lam[t] = lambda_t (blocks n floats
// apart), lambda_N = grad_out.  One volume: grid z = z.
template <int R>
__global__ void __launch_bounds__(256)
gather3k_kernel(const float* __restrict__ feat, const float* __restrict__ steps, const float* __restrict__ lam,
                const float* __restrict__ grad_out, float* __restrict__ gw_out, long long n, int N, int C, int D, int H, int W,
                int f) {
    using T = Taps3<R>;
    __shared__ float tile[kSclTH + 2 * R][kSclTW + 2 * R];
    const int x0 = blockIdx.x * kSclTW, y0 = blockIdx.y * kSclTH, z = blockIdx.z;
    const int tx = threadIdx.x, ty = threadIdx.y, x = x0 + tx, y = y0 + ty;
    const bool in = x < W && y < H;
    const size_t HW = (size_t)H * W, V = (size_t)D * HW, p = in ? (size_t)z * HW + (size_t)y * W + x : 0;
    const int zs = z + (R - f);
    const bool zin = zs >= 0 && zs < D;
    const size_t zoff = zin ? (size_t)zs * HW : 0;
    float gw[T::K * T::K];
#pragma unroll
    for (int j = 0; j < T::K * T::K; ++j) gw[j] = 0.f;
    for (int c = 0; c < C; ++c) {
        for (int t = 0; t < N; ++t) {
            const float* src = (t == 0 ? feat : steps + (size_t)(t - 1) * n) + (size_t)c * V + zoff;
            __syncthreads();
            for (int i = ty * kSclTW + tx; i < (kSclTH + 2 * R) * (kSclTW + 2 * R); i += kSclTW * kSclTH) {
                const int r = i / (kSclTW + 2 * R), q = i % (kSclTW + 2 * R);
                const int gy = y0 - R + r, gx = x0 - R + q;
                tile[r][q] = zin && gy >= 0 && gy < H && gx >= 0 && gx < W ? __ldg(src + (size_t)gy * W + gx) : 0.f;
            }
            __syncthreads();
            if (!in || !zin) continue;
            const float lp = __ldg((t == N - 1 ? grad_out : lam + (size_t)(t + 1) * n) + (size_t)c * V + p);
#pragma unroll
            for (int tt = 0; tt < T::K; ++tt)
#pragma unroll
                for (int l = 0; l < T::K; ++l) {
                    const int yy = y + R - tt, xx = x + R - l;   // taps outside the volume take no gradient
                    if (yy >= 0 && yy < H && xx >= 0 && xx < W) gw[tt * T::K + l] = fmaf(lp, tile[ty + 2 * R - tt][tx + 2 * R - l], gw[tt * T::K + l]);
                }
        }
    }
    if (!in) return;
#pragma unroll
    for (int tt = 0; tt < T::K; ++tt)
#pragma unroll
        for (int l = 0; l < T::K; ++l) {
            if (tt == R && l == R && f == R) continue;
            gw_out[(size_t)T::tap(f, tt, l) * V + p] = gw[tt * T::K + l];
        }
}

// The chain rule.  Gathered (mode 0/1): w_k = a_k / S with S = sum_j |a_j|, kappa = 1 - sum_k w_k, so with
// Gkappa = sum_c Gc_c d0_c, H_k = Gw_k - Gkappa and T = sum_k H_k w_k:  dL/da_j = (H_j - sign(a_j) T) / S.  'paddle'
// (mode 2): no centre term, H_k = Gw_k.  wk holds Gw_0..Gw_{NT-1} and kappa; Gc_c = sum_t lambda_{t+1,c} is summed here.
// Gathered: grad_g_j lands at p + off_j (each g_j(q) feeds one voxel: no atomics), grad_feat = kappa Gc + lambda_0.  'paddle': grad_g_j lands at p, grad_feat = lambda_0.  One volume: grid z = z.
template <int R>
__global__ void __launch_bounds__(256)
fin3k_kernel(const float* __restrict__ g, const float* __restrict__ feat, const float* __restrict__ wk,
             const float* __restrict__ lam, const float* __restrict__ grad_out, float* __restrict__ grad_g,
             float* __restrict__ grad_feat, long long n, int N, int C, int D, int H, int W, int mode) {
    using T = Taps3<R>;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    const int z = blockIdx.z;
    if (x >= W || y >= H) return;
    const size_t V = (size_t)D * H * W, p = ((size_t)z * H + y) * W + x;
    const float kappa = __ldg(wk + T::NT * V + p);
    float gkappa = 0.f;
    for (int c = 0; c < C; ++c) {
        const size_t q = (size_t)c * V + p;
        float gc = 0.f;
        for (int t = 0; t < N; ++t) gc += __ldg((t == N - 1 ? grad_out : lam + (size_t)(t + 1) * n) + q);
        gkappa = fmaf(gc, __ldg(feat + q), gkappa);
        if (grad_feat) grad_feat[q] = mode == 2 ? __ldg(lam + q) : fmaf(kappa, gc, __ldg(lam + q));
    }
    if (!grad_g) return;
    if (mode == 2) gkappa = 0.f;   // no centre term
    float S = 0.f;
#pragma unroll 4
    for (int k = 0; k < T::NT; ++k) S += fabsf(prep_tap<R>(g, k, z, y, x, D, H, W, V, p, mode));
    float Tsum = 0.f;
#pragma unroll 4
    for (int k = 0; k < T::NT; ++k)
        Tsum = fmaf(__ldg(wk + k * V + p) - gkappa, __fdiv_rn(prep_tap<R>(g, k, z, y, x, D, H, W, V, p, mode), S), Tsum);
#pragma unroll 4
    for (int k = 0; k < T::NT; ++k) {
        const float hk = __ldg(wk + k * V + p) - gkappa;
        if (mode == 2) {
            const float v = __ldg(g + k * V + p);
            grad_g[k * V + p] = __fdiv_rn(hk - signf(fabsf(v)) * Tsum, S) * signf(v);
        } else {
            const int zz = z + T::dz(k), yy = y + T::dy(k), xx = x + T::dx(k);
            if (!inside3(zz, yy, xx, D, H, W)) continue;
            const size_t q = ((size_t)zz * H + yy) * W + xx;
            const float v = __ldg(g + k * V + q);
            const float a = mode == 1 ? fabsf(v) : v;
            // d|g|/dg = sign(g) (0 at 0, like torch.abs) in the _abs norm
            grad_g[k * V + q] = __fdiv_rn(hk - signf(a) * Tsum, S) * (mode == 1 ? signf(v) : 1.f);
        }
    }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// RAW: w is the caller's gates (the step with PADDLE false and RAW true); otherwise `paddle` picks the PADDLE mode
template <int R, bool RAW, bool FAN>
void launch_step_as(bool vec, bool paddle, const float* w, const float* d0, const float* cur, float* dst, int nbc, int C, int D,
                    int H, int W, cudaStream_t s, const Fan& fan) {
    const unsigned gz = (unsigned)(D * nbc);
    if (vec) {
        const dim3 grid((W + kVecTW - 1) / kVecTW, (H + kVecTH - 1) / kVecTH, gz), block(16, 16);
        if constexpr (RAW) step3k_vec_kernel<R, false, true, FAN><<<grid, block, 0, s>>>(w, nullptr, cur, dst, C, D, H, W, fan);
        else if (paddle) step3k_vec_kernel<R, true, false, FAN><<<grid, block, 0, s>>>(w, d0, cur, dst, C, D, H, W, fan);
        else step3k_vec_kernel<R, false, false, FAN><<<grid, block, 0, s>>>(w, d0, cur, dst, C, D, H, W, fan);
    } else {
        const dim3 grid((W + kSclTW - 1) / kSclTW, (H + kSclTH - 1) / kSclTH, gz), block(kSclTW, kSclTH);
        if constexpr (RAW) step3k_scalar_kernel<R, false, true, FAN><<<grid, block, 0, s>>>(w, nullptr, cur, dst, C, D, H, W, fan);
        else if (paddle) step3k_scalar_kernel<R, true, false, FAN><<<grid, block, 0, s>>>(w, d0, cur, dst, C, D, H, W, fan);
        else step3k_scalar_kernel<R, false, false, FAN><<<grid, block, 0, s>>>(w, d0, cur, dst, C, D, H, W, fan);
    }
}

// fan non-null: the FAN instantiation, which also stores the result to fan's destinations
template <int R, bool RAW = false>
void launch_step(bool vec, bool paddle, const float* w, const float* d0, const float* cur, float* dst, int nbc, int C, int D,
                 int H, int W, cudaStream_t s, const Fan* fan = nullptr) {
    if (fan) launch_step_as<R, RAW, true>(vec, paddle, w, d0, cur, dst, nbc, C, D, H, W, s, *fan);
    else launch_step_as<R, RAW, false>(vec, paddle, w, d0, cur, dst, nbc, C, D, H, W, s, Fan{});
}

// fan (fused gather): destinations addressed like out, which the last step of every launch group also writes, each offset
// to the group as `out` is
template <int R>
int forward_3k(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int iters, int mode,
               void* ws, cudaStream_t stream, int* launches, const Fan* fan) {
    using T = Taps3<R>;
    const size_t V = (size_t)D * H * W, n = (size_t)C * V;
    const int G = group3d(B, C, D, H, W, iters, T::NP);
    float* wk = static_cast<float*>(ws);          // [G][NP][V]
    float* tmp = wk + (size_t)G * T::NP * V;      // [G][C][V]
    const bool vec = W % 4 == 0 && aligned16(guidance) && aligned16(feat) && aligned16(out) && aligned16(ws);
    const bool paddle = mode == 2;
    for (int b0 = 0; b0 < B; b0 += G) {
        const int nvol = B - b0 < G ? B - b0 : G;
        const float* g = guidance + (size_t)b0 * T::NT * V;
        const float* d0 = feat + (size_t)b0 * n;
        float* o = out + (size_t)b0 * n;
        if (!paddle) {
            prep3k_kernel<R><<<dim3((W + 31) / 32, (H + 7) / 8, D * nvol), dim3(32, 8), 0, stream>>>(g, wk, D, H, W, mode);
            ++*launches;
        }
        const Fan gfan = fan ? offset_fan(*fan, (size_t)b0 * n) : Fan{};
        const float* cur = d0;
        float* dst = (iters & 1) ? o : tmp;   // ping-pong so that the last step writes out
        for (int it = 0; it < iters; ++it) {
            launch_step<R>(vec, paddle, paddle ? g : wk, paddle ? nullptr : d0, cur, dst, nvol * C, C, D, H, W, stream,
                           fan && it == iters - 1 ? &gfan : nullptr);
            ++*launches;
            cur = dst;
            dst = (dst == o) ? tmp : o;
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

template <int R>
int backward_3k(const float* guidance, const float* feat, const float* grad_out, float* grad_g, float* grad_feat, int B, int C,
                int D, int H, int W, int iters, int mode, void* ws, cudaStream_t stream, int* launches) {
    using T = Taps3<R>;
    const size_t V = (size_t)D * H * W, n = (size_t)C * V;
    float* wk = static_cast<float*>(ws);                // [NP][V]: w_k and kappa, then Gw_k and kappa
    float* steps = wk + (size_t)T::NP * V;              // steps[t] = d_{t+1}, t < N-1
    float* lam = steps + (size_t)(iters - 1) * n;       // lam[t]   = lambda_t, t < N
    const bool vec = W % 4 == 0 && aligned16(feat) && aligned16(ws);
    const dim3 block(kSclTW, kSclTH), grid((W + kSclTW - 1) / kSclTW, (H + kSclTH - 1) / kSclTH, D);
    for (int b = 0; b < B; ++b) {
        const float* g = guidance + (size_t)b * T::NT * V;
        const float* d0 = feat + (size_t)b * n;
        const float* go = grad_out + (size_t)b * n;
        prep3k_kernel<R><<<grid, block, 0, stream>>>(g, wk, D, H, W, mode);
        ++*launches;
        for (int t = 0; t + 1 < iters; ++t) {           // d_{t+1} = step(d_t); the weight planes of 'paddle' have no kappa term
            launch_step<R>(vec, false, wk, mode == 2 ? nullptr : d0, t == 0 ? d0 : steps + (size_t)(t - 1) * n,
                           steps + (size_t)t * n, C, C, D, H, W, stream);
            ++*launches;
        }
        for (int t = iters - 1; t >= 0; --t) {          // lambda_t from lambda_{t+1}
            adj3k_kernel<R><<<dim3(grid.x, grid.y, D * C), block, 0, stream>>>(
                wk, t == iters - 1 ? go : lam + (size_t)(t + 1) * n, lam + (size_t)t * n, D, H, W);
            ++*launches;
        }
        if (grad_g) {
            for (int f = 0; f < T::K; ++f) {            // Gw over the dead weight planes, one z-slab of taps per launch
                gather3k_kernel<R><<<grid, block, 0, stream>>>(d0, steps, lam, go, wk, (long long)n, iters, C, D, H, W, f);
                ++*launches;
            }
        }
        fin3k_kernel<R><<<grid, block, 0, stream>>>(g, d0, wk, lam, go, grad_g ? grad_g + (size_t)b * T::NT * V : nullptr,
                                                    grad_feat ? grad_feat + (size_t)b * n : nullptr, (long long)n, iters, C,
                                                    D, H, W, mode);
        ++*launches;
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// ---- caller-supplied gates --------------------------------------------------------------------------------------
// Volumes per launch group: those of the paths above with no weight planes; one step needs no ping-pong buffer, so then
// only gridDim.z bounds the group.
int gates_group(int B, int C, int D, int H, int W, int iters) {
    if (iters > 1) return group3d(B, C, D, H, W, iters, 0);
    const long long gz = 65535 / ((long long)D * C);
    return (int)(gz < 1 ? 1 : (gz < B ? gz : B));
}

// fan: as in forward_3k
template <int R>
int forward_gates_3k(const float* gates, const float* feat, float* out, int B, int C, int D, int H, int W, int iters, void* ws,
                     cudaStream_t stream, int* launches, const Fan* fan) {
    using T = Taps3<R>;
    const size_t V = (size_t)D * H * W, n = (size_t)C * V;
    const int G = gates_group(B, C, D, H, W, iters);
    float* tmp = static_cast<float*>(ws);   // [G][C][V] when iters > 1
    const bool vec = W % 4 == 0 && aligned16(gates) && aligned16(feat) && aligned16(out) && aligned16(ws);
    for (int b0 = 0; b0 < B; b0 += G) {
        const int nvol = B - b0 < G ? B - b0 : G;
        const float* g = gates + (size_t)b0 * T::NT * V;
        float* o = out + (size_t)b0 * n;
        const Fan gfan = fan ? offset_fan(*fan, (size_t)b0 * n) : Fan{};
        const float* cur = feat + (size_t)b0 * n;
        float* dst = (iters & 1) ? o : tmp;   // ping-pong so that the last step writes out
        for (int it = 0; it < iters; ++it) {
            launch_step<R, true>(vec, false, g, nullptr, cur, dst, nvol * C, C, D, H, W, stream,
                                 fan && it == iters - 1 ? &gfan : nullptr);
            ++*launches;
            cur = dst;
            dst = (dst == o) ? tmp : o;
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// One volume at a time: N-1 forward steps keep d_1..d_{N-1}, N adjoint steps on the gates keep lambda_1..lambda_{N-1} and
// write lambda_0 = grad_feat, and the K gather launches write Gw_k = grad_gates.  Workspace (2N-2)*C*V floats.  Without
// grad_g the forward steps and the gathers, which only feed it, are skipped; without grad_feat the last adjoint is.
template <int R>
int backward_gates_3k(const float* gates, const float* feat, const float* grad_out, float* grad_g, float* grad_feat, int B, int C,
                      int D, int H, int W, int iters, void* ws, cudaStream_t stream, int* launches) {
    using T = Taps3<R>;
    const size_t V = (size_t)D * H * W, n = (size_t)C * V;
    float* steps = static_cast<float*>(ws);                         // steps[t] = d_{t+1}, t < N-1
    float* lam = steps + (size_t)(iters >= 2 ? iters - 2 : 0) * n;   // lam + t*n = lambda_t for 1 <= t < N (after steps)
    const bool vec = W % 4 == 0 && aligned16(gates) && aligned16(feat) && aligned16(ws);
    const dim3 block(kSclTW, kSclTH), grid((W + kSclTW - 1) / kSclTW, (H + kSclTH - 1) / kSclTH, D);
    for (int b = 0; b < B; ++b) {
        const float* g = gates + (size_t)b * T::NT * V;
        const float* d0 = feat + (size_t)b * n;
        const float* go = grad_out + (size_t)b * n;
        for (int t = 0; grad_g && t + 1 < iters; ++t) {   // d_{t+1} = step(d_t)
            launch_step<R, true>(vec, false, g, nullptr, t == 0 ? d0 : steps + (size_t)(t - 1) * n, steps + (size_t)t * n, C, C,
                                 D, H, W, stream);
            ++*launches;
        }
        for (int t = iters - 1; t >= 0; --t) {          // lambda_t from lambda_{t+1}; lambda_0 is grad_feat
            float* lout = t == 0 ? (grad_feat ? grad_feat + (size_t)b * n : nullptr) : lam + (size_t)t * n;
            if (!lout) continue;
            adj3k_kernel<R><<<dim3(grid.x, grid.y, D * C), block, 0, stream>>>(
                g, t == iters - 1 ? go : lam + (size_t)(t + 1) * n, lout, D, H, W);
            ++*launches;
        }
        if (grad_g) {
            for (int f = 0; f < T::K; ++f) {            // Gw_k = grad_g_k, one z-slab of taps per launch
                gather3k_kernel<R><<<grid, block, 0, stream>>>(d0, steps, lam, go, grad_g + (size_t)b * T::NT * V, (long long)n, iters,
                                                               C, D, H, W, f);
                ++*launches;
            }
        }
    }
    CSPN_CUDA_TRY(cudaGetLastError());
    return CSPN_OK;
}

// K = 3 -> R = 1, K = 5 -> R = 2: f(R) as an integral constant (the normalised forward exists for R = 2 only)
template <class F>
int with_radius(int K, F&& f) {
    return K == 3 ? f(std::integral_constant<int, 1>{}) : f(std::integral_constant<int, 2>{});
}

const char* name_of(Family family) { return family == Family::Gates ? " gates" : ""; }   // follows "KxKxK 3D" in messages

// The workspace holds what `need` says (nothing, for one step on the caller's gates), and the launch grids take the problem
int check_launch(int C, int D, int H, int K, Family family, const char* what, size_t need, const void* ws, size_t ws_bytes) {
    if (need && (!ws || ws_bytes < need)) {
        set_error("%dx%dx%d 3D%s %s needs %zu workspace bytes, got %zu", K, K, K, name_of(family), what, need, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    if ((long long)D * C > 65535) {
        set_error("%dx%dx%d 3D%s %s: D*C=%lld exceeds gridDim.z", K, K, K, name_of(family), what, (long long)D * C);
        return CSPN_ERR_UNSUPPORTED;
    }
    if ((H + kSclTH - 1) / kSclTH > 65535) {
        set_error("%dx%dx%d 3D%s %s: H=%d exceeds gridDim.y", K, K, K, name_of(family), what, H);
        return CSPN_ERR_UNSUPPORTED;
    }
    return CSPN_OK;
}

}  // namespace

// Normalised (every mode): K^3 weight planes and, past one step, the ping-pong buffer per volume of a group.  Gates: the
// caller's gates are the weight planes.
size_t widek3d_workspace_bytes(int B, int C, int D, int H, int W, int K, int iters, Family family) {
    if (iters <= 0) return 0;
    const size_t V = (size_t)D * H * W, np = (size_t)K * K * K;
    if (family == Family::Gates) return iters > 1 ? sizeof(float) * (size_t)gates_group(B, C, D, H, W, iters) * C * V : 0;
    return sizeof(float) * (size_t)group3d(B, C, D, H, W, iters, (int)np) * (np * V + (iters > 1 ? (size_t)C * V : 0));
}

// One volume at a time: the weight planes, d_1..d_{N-1} and every lambda_t; gates keep no weight planes and no lambda_0
size_t widek3d_bwd_workspace_bytes(int C, int D, int H, int W, int K, int iters, Family family) {
    if (iters <= 0) return 0;
    const size_t V = (size_t)D * H * W;
    if (family == Family::Gates) return sizeof(float) * (2 * (size_t)iters - 2) * C * V;
    return sizeof(float) * ((size_t)K * K * K * V + (2 * (size_t)iters - 1) * C * V);
}

int widek3d_forward(const float* guidance, const float* feat, float* out, int B, int C, int D, int H, int W, int K, int iters,
                    Family family, int mode, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, const Fan* fan) {
    if (iters == 0) {
        CSPN_CUDA_TRY(cudaMemcpyAsync(out, feat, (size_t)B * C * D * H * W * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const int rc = check_launch(C, D, H, K, family, "path", widek3d_workspace_bytes(B, C, D, H, W, K, iters, family), ws, ws_bytes);
    if (rc != CSPN_OK) return rc;
    if (family != Family::Gates) return forward_3k<2>(guidance, feat, out, B, C, D, H, W, iters, mode, ws, stream, launches, fan);
    return with_radius(K, [&](auto R) {
        return forward_gates_3k<R()>(guidance, feat, out, B, C, D, H, W, iters, ws, stream, launches, fan);
    });
}

int widek3d_backward(const float* guidance, const float* feat, const float* grad_out, float* grad_g, float* grad_feat, int B, int C,
                     int D, int H, int W, int K, int iters, Family family, int mode, void* ws, size_t ws_bytes,
                     cudaStream_t stream, int* launches) {
    const bool gates = family == Family::Gates;
    const size_t V = (size_t)D * H * W;
    // gathered norms: guidance values that no voxel reads get zero gradient.  Every gate gradient is written by the gathers
    // (g_k(p) feeds voxel p alone; a tap that reads the padding gets 0), so gates need the fill for the identity only
    if (grad_g && (!gates || iters == 0))
        CSPN_CUDA_TRY(cudaMemsetAsync(grad_g, 0, (size_t)B * (K * K * K - 1) * V * sizeof(float), stream));
    if (iters == 0) {   // the identity: no dependence on the guidance
        if (grad_feat) CSPN_CUDA_TRY(cudaMemcpyAsync(grad_feat, grad_out, (size_t)B * C * V * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return CSPN_OK;
    }
    const int rc = check_launch(C, D, H, K, family, "backward", widek3d_bwd_workspace_bytes(C, D, H, W, K, iters, family), ws, ws_bytes);
    if (rc != CSPN_OK) return rc;
    if (gates && !grad_g && !grad_feat) return CSPN_OK;
    return with_radius(K, [&](auto R) {
        if (!gates) return backward_3k<R()>(guidance, feat, grad_out, grad_g, grad_feat, B, C, D, H, W, iters, mode, ws, stream, launches);
        return backward_gates_3k<R()>(guidance, feat, grad_out, grad_g, grad_feat, B, C, D, H, W, iters, ws, stream, launches);
    });
}

}  // namespace cspn
