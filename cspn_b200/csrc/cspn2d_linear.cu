// Linear spatial propagation with three-way connections: SPN's scans (Liu et al., NIPS 2017; DESIGN.md section 4.24).
// feat x (B, C, H, W) is scanned in each requested direction d of l2r, r2l, t2b, b2t (mask bits 1, 2, 4, 8, canonical
// order).  For l2r the scan index t is the column and the lateral index i the row; a step reads the previous column at
// rows i - 1, i, i + 1:
//
//   c      = ((1 - g0) - g1) - g2                                      (each subtraction rounded on its own)
//   h[i,t] = fma(g2, h[i+1,t-1], fma(g1, h[i,t-1], fma(g0, h[i-1,t-1], c * x[i,t])))      (c * x one rounded product)
//
// with g_j = gate_j[i,t] at the current node, as given.  A read outside the image is 0.  r2l reads column t + 1, t2b and
// b2t scan rows and read row y -+ 1 at columns x - 1, x, x + 1; tap j is always lateral offset j - 1 along increasing
// index, and every direction uses the same order, so each is an exact transpose and / or flip of l2r.  The gates are
// (B, 3*nd*Cg, H, W), Cg = 1 (shared by the C channels) or C (per channel): direction block k (the k-th requested
// direction) is channels [3k*Cg, 3(k+1)*Cg) and channel c uses 3c .. 3c+2 within it.
//
// Merge (nd > 1): out = h_{d*}, d* the first requested direction whose h is NaN, else the first attaining the maximum
// (torch.stack(hs).max(0)).
//
// Backward, over the saved planes, the adjoint scan in reverse scan order with delta the total adjoint of h and "n" the
// next node in scan order (t + 1 for l2r; all zero past the last node and outside the lateral range):
//   delta[i,t] = fma(g2n[i-1], deltan[i-1], fma(g1n[i], deltan[i], fma(g0n[i+1], deltan[i+1], go_d[i,t])))
//   go_d       = grad_out where d = d*, else +0                           (d* recomputed from the saved planes)
//   grad_x_d   = c * delta,        grad_g_j = delta * (h_nb_j - x)        (h_nb_j = h[i+j-1, t-1], 0 outside; the
//                                                                           difference and the product rounded apart)
//   grad_x     = ((grad_x_0 + grad_x_1) + grad_x_2) + grad_x_3            (requested directions in canonical order)
//   shared gates: grad_g = sum over c ascending, starting from c = 0's value
// No atomics and no memsets: every output word is written by one thread.
//
// Kernels (sm_90a):
//   scan      one launch for all requested directions, grid (CS * B*C, nd) in clusters of CS CTAs.  The CS CTAs of a
//             cluster split the lateral axis of one plane and direction into segments of Lseg lanes.  Each CTA scans
//             a window of its segment plus a kHalo-lane halo on each side, one thread per window lane, in chunks of
//             kHalo steps.  The dependency cone widens by one lane per step, so after a chunk the segment's lanes are
//             exact and the halo lanes are not; the CTAs then publish their segment's last row in shared memory, pass
//             one cluster barrier, and read the halo lanes of the next chunk from the owning CTAs over DSMEM.  The
//             halo lanes repeat the segment's arithmetic on the same inputs, so the plan changes no bit.  Within a
//             chunk the lanes exchange through a double-buffered shared row, one __syncthreads per step.
//             x, the gates (the backward also: the routed grad_out and the saved plane) are staged per chunk in shared
//             memory by cp.async, double-buffered: the next chunk's copies are issued before the current chunk is
//             scanned.  One staging loop serves both orientations: the copies run along memory (steps for l2r / r2l,
//             lanes for t2b / b2t) and only the shared-memory index transposes.  h (the backward's gradients) is
//             collected in shared memory and written back per chunk in the same memory order.
//   pick      the per-pixel selection: forward out; backward the routed grad_out of every direction.
//   finalize  the direction sum of grad_x and the channel sum of a shared gate's gradient, each output word by one thread.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cspn {
namespace {

namespace cg = cooperative_groups;

constexpr int kHalo = 8;                             // halo lanes per side = steps per chunk
constexpr int kLinMaxSeg = 256;                      // lanes per segment
constexpr int kLinMaxCluster = 8;                    // CTAs per cluster (the portable limit)
constexpr int kLinMaxLateral = kLinMaxSeg * kLinMaxCluster;
constexpr int kLinThreads = (kLinMaxSeg + 2 * kHalo + 31) / 32 * 32;   // one thread per window lane, whole warps
constexpr int kLinTargetCtas = 264;                 // a cluster split is chosen while the grid has fewer CTAs than this
constexpr int kLinMergeThreads = 256;
constexpr int kLinMergeBlocks = 16 * 132;            // grid-stride cap of the per-pixel passes

// the canonical direction (0 l2r, 1 r2l, 2 t2b, 3 b2t) of the k-th set bit of mask
__device__ __forceinline__ int kth_dir(int mask, int k) {
    int d = 0;
    for (; d < 4; ++d)
        if ((mask >> d) & 1) {
            if (k == 0) break;
            --k;
        }
    return d;
}

// The geometry of a scan in direction d over an H x W plane: lanes L, steps S, the element offset of (lane, step s)
struct Scan {
    int L, S;
    size_t lstr, tstr;
    bool rev, horiz;
    __device__ Scan(int d, int H, int W)
        : L(d < 2 ? H : W), S(d < 2 ? W : H), lstr(d < 2 ? (size_t)W : 1), tstr(d < 2 ? 1 : (size_t)W), rev(d & 1), horiz(d < 2) {}
    __device__ size_t at(int lane, int s) const { return (size_t)lane * lstr + (size_t)(rev ? S - 1 - s : s) * tstr; }
};

__device__ __forceinline__ void cp4(float* dst, const float* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Stages `rows` rows of a plane into dst[r * pitch + 1 + w] for the window lanes w in [0, Wn) (lane = lane0 + w); row r
// holds step s0 + dir * r.  Outside the plane (lane or step) the copy fills 0.  The copies run along memory: steps
// innermost for a horizontal scan, lanes for a vertical one.
__device__ __forceinline__ void stage(float* dst, int pitch, const float* plane, const Scan& sc, int lane0, int Wn, int rows, int s0,
                                      int dir) {
    const int n = rows * Wn;
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int w = sc.horiz ? idx / rows : idx % Wn, r = sc.horiz ? idx % rows : idx / Wn;
        const int lane = lane0 + w, s = s0 + dir * r;
        const bool in = lane >= 0 && lane < sc.L && s >= 0 && s < sc.S;
        cp4(dst + r * pitch + 1 + w, plane + (in ? sc.at(lane, s) : 0), in);
    }
}

// Writes src[r * pitch + o] (rows r < rows, segment lanes o < own) to the plane at (lane0 + o, s0 + dir * r), in memory
// order as stage() reads
__device__ __forceinline__ void unstage(float* plane, const float* src, int pitch, const Scan& sc, int lane0, int own, int rows,
                                        int s0, int dir) {
    const int n = rows * own;
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int o = sc.horiz ? idx / rows : idx % own, r = sc.horiz ? idx % rows : idx / own;
        plane[sc.at(lane0 + o, s0 + dir * r)] = src[r * pitch + o];
    }
}

// Reads the halo lanes of the window (w < kHalo or w >= kHalo + own) from the CTAs that own them: pub of rank q holds
// its segment's lanes [q * Lseg, (q + 1) * Lseg).  Lanes outside the plane are 0.
__device__ __forceinline__ void read_halo(cg::cluster_group& cl, float* row, const float* pub, int a, int Lseg, int own, int Wn, int L) {
    const int w = threadIdx.x;
    if (w < Wn && (w < kHalo || w >= kHalo + own)) {
        const int lane = a - kHalo + w;
        float v = 0.f;
        if (lane >= 0 && lane < L) {
            const int q = lane / Lseg;
            v = cl.map_shared_rank(const_cast<float*>(pub), q)[lane - q * Lseg];
        }
        row[w + 1] = v;
    }
}

// Shared memory of a scan CTA, in floats, for window pitch P = Lseg_max + 2*kHalo + 2 (pads included)
__host__ __device__ constexpr int fwd_smem_floats(int P, int seg) { return 2 * 4 * kHalo * P + 2 * P + kHalo * seg + 2 * seg; }
__host__ __device__ constexpr int bwd_smem_floats(int P, int seg) {
    return 2 * (kHalo + 3 * (kHalo + 1) + 2 * kHalo) * P + 2 * P + 4 * kHalo * seg + 2 * seg;
}

struct LinGeom {
    int CS, seg_h, seg_v, seg, P;                    // cluster size, segment lanes per orientation, their max, window pitch
};

__global__ void __launch_bounds__(kLinThreads, 1)
lin_fwd_kernel(const float* __restrict__ feat, const float* __restrict__ gate, float* __restrict__ planes, int C, int H, int W, int mask,
               int Cg, LinGeom geo) {
    extern __shared__ __align__(16) float sm[];
    cg::cluster_group cl = cg::this_cluster();
    const int P = geo.P, seg = geo.seg;
    float* st = sm;                                  // [2][4][kHalo][P]: x, g0, g1, g2 per chunk
    float* row = st + 2 * 4 * kHalo * P;             // [2][P]: h of the previous step by window lane + 1
    float* hout = row + 2 * P;                       // [kHalo][seg]
    float* pub = hout + kHalo * seg;                 // [2][seg]: the segment's last row, per chunk parity
    const int tid = threadIdx.x, rank = (int)cl.block_rank(), bc = blockIdx.x / geo.CS, k = blockIdx.y, nd = __popc(mask);
    const size_t HW = (size_t)H * W, P_all = (size_t)(gridDim.x / geo.CS) * HW;
    const Scan sc(kth_dir(mask, k), H, W);
    const int Lseg = sc.horiz ? geo.seg_h : geo.seg_v, Wn = Lseg + 2 * kHalo, a = rank * Lseg;
    const int own = max(0, min(Lseg, sc.L - a)), lane0 = a - kHalo;
    const int b = bc / C, c = bc - b * C;
    const float* x = feat + (size_t)bc * HW;
    const float* g = gate + ((size_t)b * 3 * nd * Cg + 3 * ((size_t)k * Cg + (Cg > 1 ? c : 0))) * HW;
    float* h = planes + (size_t)k * P_all + (size_t)bc * HW;
    for (int q = tid; q < 2 * P; q += blockDim.x) row[q] = 0.f;

    auto issue = [&](int ch) {
        float* s = st + (ch & 1) * 4 * kHalo * P;
        const int s0 = ch * kHalo;
        stage(s, P, x, sc, lane0, Wn, kHalo, s0, 1);
        for (int j = 0; j < 3; ++j) stage(s + (1 + j) * kHalo * P, P, g + j * HW, sc, lane0, Wn, kHalo, s0, 1);
        cp_commit();
    };
    const int nch = (sc.S + kHalo - 1) / kHalo;
    issue(0);
    int cur = 0;
    const int w = tid, lane = lane0 + w;
    const bool live = w < Wn && lane >= 0 && lane < sc.L, mine = w >= kHalo && w < kHalo + own;
    for (int ch = 0; ch < nch; ++ch) {
        if (ch + 1 < nch) {
            issue(ch + 1);
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        const float* s = st + (ch & 1) * 4 * kHalo * P;
        const int s0 = ch * kHalo, nq = min(kHalo, sc.S - s0);
        for (int q = 0; q < nq; ++q) {
            if (live) {
                const float* rp = row + cur * P;
                const float xv = s[q * P + w + 1], g0 = s[(kHalo + q) * P + w + 1], g1 = s[(2 * kHalo + q) * P + w + 1],
                            g2 = s[(3 * kHalo + q) * P + w + 1];
                const float cc = __fsub_rn(__fsub_rn(__fsub_rn(1.f, g0), g1), g2);
                const float v = fmaf(g2, rp[w + 2], fmaf(g1, rp[w + 1], fmaf(g0, rp[w], __fmul_rn(cc, xv))));
                row[(cur ^ 1) * P + w + 1] = v;
                if (mine) hout[q * seg + w - kHalo] = v;
            }
            __syncthreads();
            cur ^= 1;
        }
        if (mine) pub[(ch & 1) * seg + w - kHalo] = row[cur * P + w + 1];
        unstage(h, hout, seg, sc, a, own, nq, s0, 1);
        cl.sync();                                   // the published rows are complete; hout may be refilled
        read_halo(cl, row + cur * P, pub + (ch & 1) * seg, a, Lseg, own, Wn, sc.L);
    }
    cl.sync();                                       // no CTA leaves while another reads its shared memory
}

// The adjoint scan of direction block k = blockIdx.y over the saved plane, from the last step backwards.  god: the routed
// grad_out of this direction (grad_out itself for nd = 1, else the pick's planes [k][B*C][HW]).  gx: grad_x's plane of
// this direction (grad_feat itself for nd = 1, else a partial plane [k][B*C][HW]) or null.  gg: grad_gate laid out as
// the gate (direct) or the partial planes [k][B*C][3][HW] (a shared gate with C > 1), or null.
__global__ void __launch_bounds__(kLinThreads, 1)
lin_bwd_kernel(const float* __restrict__ feat, const float* __restrict__ gate, const float* __restrict__ planes,
               const float* __restrict__ god, float* __restrict__ gx, float* __restrict__ gg, bool gg_direct, int C, int H, int W, int mask,
               int Cg, LinGeom geo) {
    extern __shared__ __align__(16) float sm[];
    cg::cluster_group cl = cg::this_cluster();
    const int P = geo.P, seg = geo.seg;
    constexpr int kRows = kHalo + 3 * (kHalo + 1) + 2 * kHalo;   // x, g0..g2 (one row more: the next step), go, h(s - 1)
    float* st = sm;                                  // [2][kRows][P]
    float* dl = st + 2 * kRows * P;                  // [2][P]: delta of the next step by window lane + 1
    float* outs = dl + 2 * P;                        // [4][kHalo][seg]: grad_x, grad_g0..2
    float* pub = outs + 4 * kHalo * seg;             // [2][seg]
    const int tid = threadIdx.x, rank = (int)cl.block_rank(), bc = blockIdx.x / geo.CS, k = blockIdx.y, nd = __popc(mask);
    const int BC = gridDim.x / geo.CS;
    const size_t HW = (size_t)H * W, P_all = (size_t)BC * HW;
    const Scan sc(kth_dir(mask, k), H, W);
    const int Lseg = sc.horiz ? geo.seg_h : geo.seg_v, Wn = Lseg + 2 * kHalo, a = rank * Lseg;
    const int own = max(0, min(Lseg, sc.L - a)), lane0 = a - kHalo;
    const int b = bc / C, c = bc - b * C;
    const float* x = feat + (size_t)bc * HW;
    const size_t goff = ((size_t)b * 3 * nd * Cg + 3 * ((size_t)k * Cg + (Cg > 1 ? c : 0))) * HW;
    const float* g = gate + goff;
    const float* h = planes + (size_t)k * P_all + (size_t)bc * HW;
    const float* go = god + (nd > 1 ? (size_t)k * P_all : 0) + (size_t)bc * HW;
    float* gxo = gx ? gx + (nd > 1 ? (size_t)k * P_all : 0) + (size_t)bc * HW : nullptr;
    float* ggo = gg ? gg + (gg_direct ? goff : ((size_t)k * BC + bc) * 3 * HW) : nullptr;
    for (int q = tid; q < 2 * kRows * P + 2 * P; q += blockDim.x) sm[q] = 0.f;     // the stage's pads stay 0
    __syncthreads();

    // chunk ch covers steps s1 - q, q < kHalo, s1 = S - 1 - ch*kHalo; rows: x [0, K), g_j [K + j(K+1), ...) from step
    // s1 + 1 down, go [4K + 3, ...), h(s - 1) after it
    constexpr int rG = kHalo, rGO = kHalo + 3 * (kHalo + 1), rH = rGO + kHalo;
    auto issue = [&](int ch) {
        float* s = st + (ch & 1) * kRows * P;
        const int s1 = sc.S - 1 - ch * kHalo;
        stage(s, P, x, sc, lane0, Wn, kHalo, s1, -1);
        for (int j = 0; j < 3; ++j) stage(s + (rG + j * (kHalo + 1)) * P, P, g + j * HW, sc, lane0, Wn, kHalo + 1, s1 + 1, -1);
        stage(s + rGO * P, P, go, sc, lane0, Wn, kHalo, s1, -1);
        stage(s + rH * P, P, h, sc, lane0, Wn, kHalo, s1 - 1, -1);
        cp_commit();
    };
    const int nch = (sc.S + kHalo - 1) / kHalo;
    issue(0);
    int cur = 0;
    const int w = tid, lane = lane0 + w;
    const bool live = w < Wn && lane >= 0 && lane < sc.L, mine = w >= kHalo && w < kHalo + own;
    for (int ch = 0; ch < nch; ++ch) {
        if (ch + 1 < nch) {
            issue(ch + 1);
            cp_wait<1>();
        } else {
            cp_wait<0>();
        }
        __syncthreads();
        const float* s = st + (ch & 1) * kRows * P;
        const float* G0 = s + rG * P;
        const float* G1 = G0 + (kHalo + 1) * P;
        const float* G2 = G1 + (kHalo + 1) * P;
        const int s1 = sc.S - 1 - ch * kHalo, nq = min(kHalo, s1 + 1);
        for (int q = 0; q < nq; ++q) {
            if (live) {
                const float* dp = dl + cur * P;
                const float del = fmaf(G2[q * P + w], dp[w],
                                       fmaf(G1[q * P + w + 1], dp[w + 1], fmaf(G0[q * P + w + 2], dp[w + 2], s[(rGO + q) * P + w + 1])));
                dl[(cur ^ 1) * P + w + 1] = del;
                if (mine) {
                    const int o = q * seg + w - kHalo;
                    const float g0 = G0[(q + 1) * P + w + 1], g1 = G1[(q + 1) * P + w + 1], g2 = G2[(q + 1) * P + w + 1];
                    const float xv = s[q * P + w + 1];
                    const float* hp = s + (rH + q) * P + w;
                    outs[o] = __fmul_rn(__fsub_rn(__fsub_rn(__fsub_rn(1.f, g0), g1), g2), del);
                    outs[kHalo * seg + o] = __fmul_rn(del, __fsub_rn(hp[0], xv));
                    outs[2 * kHalo * seg + o] = __fmul_rn(del, __fsub_rn(hp[1], xv));
                    outs[3 * kHalo * seg + o] = __fmul_rn(del, __fsub_rn(hp[2], xv));
                }
            }
            __syncthreads();
            cur ^= 1;
        }
        if (mine) pub[(ch & 1) * seg + w - kHalo] = dl[cur * P + w + 1];
        if (gxo) unstage(gxo, outs, seg, sc, a, own, nq, s1, -1);
        if (ggo)
            for (int j = 0; j < 3; ++j) unstage(ggo + j * HW, outs + (1 + j) * kHalo * seg, seg, sc, a, own, nq, s1, -1);
        cl.sync();
        read_halo(cl, dl + cur * P, pub + (ch & 1) * seg, a, Lseg, own, Wn, sc.L);
    }
    cl.sync();
}

// d* of pixel p over the nd planes: the first NaN, else the first maximum
struct Pick {
    float v;
    int k;
};
__device__ __forceinline__ Pick merge_pick(const float* __restrict__ planes, size_t P, size_t p, int nd) {
    Pick r{__ldg(planes + p), 0};
    for (int k = 1; k < nd; ++k) {
        const float v = __ldg(planes + (size_t)k * P + p);
        if (!isnan(r.v) && (isnan(v) || v > r.v)) r = Pick{v, k};
    }
    return r;
}

// forward: out[p] = h_{d*}(p); backward: god[k][p] = grad_out[p] for k = d*, else +0
__global__ void __launch_bounds__(kLinMergeThreads)
lin_merge_kernel(const float* __restrict__ planes, float* __restrict__ out, const float* __restrict__ grad_out, float* __restrict__ god,
                 size_t P, int nd) {
    for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (size_t)gridDim.x * blockDim.x) {
        const Pick pk = merge_pick(planes, P, p, nd);
        if (out) out[p] = pk.v;
        if (god) {
            const float gv = __ldg(grad_out + p);
            for (int k = 0; k < nd; ++k) god[(size_t)k * P + p] = k == pk.k ? gv : 0.f;
        }
    }
}

// grad_x = the partial planes summed over k ascending (fx: [nd][P]); grad_gate of a shared gate = fg [nd][B*C][3][HW]
// summed over c ascending.  blockIdx.y: 0 grad_x, 1 grad_gate.
__global__ void __launch_bounds__(kLinMergeThreads)
lin_finalize_kernel(const float* __restrict__ fx, const float* __restrict__ fg, float* __restrict__ grad_x, float* __restrict__ grad_g,
                    int B, int C, size_t HW, int nd) {
    const size_t P = (size_t)B * C * HW;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    if (blockIdx.y == 0) {
        if (!grad_x) return;
        for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += stride) {
            float s = __ldg(fx + p);
            for (int k = 1; k < nd; ++k) s = __fadd_rn(s, __ldg(fx + (size_t)k * P + p));
            grad_x[p] = s;
        }
    } else {
        if (!grad_g) return;
        const size_t n = (size_t)B * nd * 3 * HW;            // grad_gate [B][nd][3][HW]
        for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
            const size_t pix = e % HW, r = e / HW;
            const int j = (int)(r % 3), k = (int)(r / 3 % nd), b = (int)(r / 3 / nd);
            const float* src = fg + (((size_t)k * B + b) * C * 3 + j) * HW + pix;
            float s = __ldg(src);
            for (int c = 1; c < C; ++c) s = __fadd_rn(s, __ldg(src + (size_t)c * 3 * HW));
            grad_g[e] = s;
        }
    }
}

int up_div(int a, int b) { return (a + b - 1) / b; }

int lateral_max(int H, int W, int mask) {
    const int lh = (mask & 3) ? H : 0, lv = (mask & 12) ? W : 0;
    return lh > lv ? lh : lv;
}

// The plan from the shape: CS CTAs per plane and direction, at least enough for segments of kLinMaxSeg lanes, and while
// the grid has fewer than kLinTargetCtas CTAs a power of two up to kLinMaxCluster, as long as a segment keeps 2*kHalo lanes
LinGeom lin_plan(int B, int C, int H, int W, int mask) {
    const int nd = __builtin_popcount(mask), L = lateral_max(H, W, mask);
    int cs = 1;
    const long long ctas = (long long)nd * B * C;
    while (cs < kLinMaxCluster && ctas * cs * 2 <= kLinTargetCtas && L / (cs * 2) >= 2 * kHalo) cs *= 2;
    cs = cs > up_div(L, kLinMaxSeg) ? cs : up_div(L, kLinMaxSeg);
    LinGeom g{};
    g.CS = cs;
    g.seg_h = (mask & 3) ? up_div(H, cs) : 0;
    g.seg_v = (mask & 12) ? up_div(W, cs) : 0;
    g.seg = g.seg_h > g.seg_v ? g.seg_h : g.seg_v;
    g.P = g.seg + 2 * kHalo + 2;
    return g;
}

int lin_threads(const LinGeom& g) { return up_div(g.seg + 2 * kHalo, 32) * 32; }

unsigned merge_blocks(size_t n) {
    const size_t blocks = (n + kLinMergeThreads - 1) / kLinMergeThreads;
    return (unsigned)(blocks < kLinMergeBlocks ? blocks : kLinMergeBlocks);
}

template <class Kern, class... Args>
int launch_scan(Kern kern, const LinGeom& geo, int BC, int nd, size_t smem, cudaStream_t st, Args... args) {
    CSPN_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(BC * geo.CS), (unsigned)nd);
    cfg.blockDim = dim3((unsigned)lin_threads(geo));
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = geo.CS;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    CSPN_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, args...));
    return CSPN_OK;
}

}  // namespace

int linear2d_launchable(int B, int C, int H, int W, int mask, const char** why) {
    if (lateral_max(H, W, mask) > kLinMaxLateral) {
        *why = "the lateral extent (H for l2r / r2l, W for t2b / b2t) exceeds 2048";
        return 0;
    }
    if ((long long)B * C * lin_plan(B, C, H, W, mask).CS > INT32_MAX) { *why = "B*C times the cluster size exceeds gridDim.x (2^31 - 1)"; return 0; }
    return 1;
}

size_t linear2d_workspace_bytes(int B, int C, int H, int W, int mask) {
    const int nd = __builtin_popcount(mask);
    return nd > 1 ? (size_t)nd * B * C * H * W * sizeof(float) : 0;
}

size_t linear2d_bwd_workspace_bytes(int B, int C, int H, int W, int mask, int Cg) {
    const int nd = __builtin_popcount(mask);
    const size_t P = (size_t)B * C * H * W;
    size_t n = 0;
    if (nd > 1) n += (size_t)2 * nd * P * sizeof(float);                         // grad_x partials, then the routed grad_out
    if (Cg == 1 && C > 1) n += (size_t)nd * 3 * P * sizeof(float);                // a shared gate's partials
    return n;
}

int linear2d_forward(const float* feat, const float* gate, float* out, float* planes, int B, int C, int H, int W, int mask, int Cg,
                     cudaStream_t st, int* launches) {
    const int nd = __builtin_popcount(mask);
    const LinGeom geo = lin_plan(B, C, H, W, mask);
    float* dst = nd > 1 ? planes : out;
    const size_t smem = (size_t)fwd_smem_floats(geo.P, geo.seg) * sizeof(float);
    const int rc = launch_scan(lin_fwd_kernel, geo, B * C, nd, smem, st, feat, gate, dst, C, H, W, mask, Cg, geo);
    if (rc != CSPN_OK) return rc;
    *launches = 1;
    if (nd > 1) {
        const size_t P = (size_t)B * C * H * W;
        lin_merge_kernel<<<merge_blocks(P), kLinMergeThreads, 0, st>>>(planes, out, nullptr, nullptr, P, nd);
        CSPN_CUDA_TRY(cudaGetLastError());
        *launches = 2;
    }
    return CSPN_OK;
}

int linear2d_backward(const float* feat, const float* gate, const float* planes, const float* grad_out, float* grad_feat,
                      float* grad_gate, int B, int C, int H, int W, int mask, int Cg, void* ws, cudaStream_t st, int* launches) {
    const int nd = __builtin_popcount(mask);
    const size_t P = (size_t)B * C * H * W, HW = (size_t)H * W;
    *launches = 0;
    if (!grad_feat && !grad_gate) return CSPN_OK;
    float* w = static_cast<float*>(ws);
    float* fx = nullptr;
    float* god = nullptr;
    if (nd > 1) {
        fx = w;
        god = w + (size_t)nd * P;
        w += (size_t)2 * nd * P;
    }
    const bool gg_direct = !(Cg == 1 && C > 1);
    float* fg = gg_direct ? nullptr : w;
    int nl = 0;
    if (nd > 1) {
        lin_merge_kernel<<<merge_blocks(P), kLinMergeThreads, 0, st>>>(planes, nullptr, grad_out, god, P, nd);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
    }
    float* gx = grad_feat ? (nd > 1 ? fx : grad_feat) : nullptr;
    float* gg = grad_gate ? (gg_direct ? grad_gate : fg) : nullptr;
    const LinGeom geo = lin_plan(B, C, H, W, mask);
    const size_t smem = (size_t)bwd_smem_floats(geo.P, geo.seg) * sizeof(float);
    const int rc = launch_scan(lin_bwd_kernel, geo, B * C, nd, smem, st, feat, gate, planes, nd > 1 ? (const float*)god : grad_out, gx,
                               gg, gg_direct, C, H, W, mask, Cg, geo);
    if (rc != CSPN_OK) return rc;
    ++nl;
    float* fin_x = grad_feat && nd > 1 ? grad_feat : nullptr;
    float* fin_g = grad_gate && !gg_direct ? grad_gate : nullptr;
    if (fin_x || fin_g) {
        const dim3 grid(merge_blocks(P), 2);
        lin_finalize_kernel<<<grid, kLinMergeThreads, 0, st>>>(fx, fg, fin_x, fin_g, B, C, HW, nd);
        CSPN_CUDA_TRY(cudaGetLastError());
        ++nl;
    }
    *launches = nl;
    return CSPN_OK;
}

}  // namespace cspn
