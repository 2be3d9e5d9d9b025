// 2D CSPN, all N iterations in ONE launch with HBM touched once per tile (sm_90a: TMA, clusters, DSMEM, mbarrier).
//
// Reference arithmetic: /root/reference/cspn_pytorch/models/cspn.py:42-144 (see cspn2d_generic.cu
// for the folded form d <- c' + sum_k w'_k shift_k(d)).
//
// Decomposition
//   task     = (image b, channel c, x-strip j).  A strip is TW = 32*PC columns wide; when the image is
//              wider than one strip, neighbouring strips overlap by a halo of N columns per side (the
//              stale region creeps inwards one column per iteration, so after N iterations the strip's
//              "useful" columns are still exact).  Rows are never tiled: zero padding at the top/bottom of
//              the image is the reference's own boundary condition, so a task always spans the full height.
//   cluster  = one task.  The CS CTAs of a thread-block cluster stack along y; CTA r owns the band of
//              RB = NW*PR rows starting at r*RB.  (CS*RB >= H.)
//   CTA      = NW warps stacked along y; warp wy owns PR rows; lane l owns PC consecutive columns.
//   thread   = a PR x PC pixel patch whose state lives in registers for all N iterations: 8 folded weights and
//              the current value per pixel (two value sets alternate as input / output of a step); the constant
//              term c' is read from shared memory once per step.
// Data movement
//   * the 8 guidance planes arrive by TMA (cp.async.bulk.tensor.3d), one box per channel whose origin is shifted
//     by that channel's dy: the ROW gather of cspn.py:105-132 is free and TMA's out-of-bounds zero fill is exactly
//     ZeroPad2d.  The column shift (dx = +-1) cannot ride on the box origin -- TMA needs a 16-byte aligned
//     innermost coordinate -- so boxes carry a 4-column apron and the shift is a shuffle in the prologue;
//   * clusters are persistent: the next task's boxes are issued as soon as the prologue has consumed the staging
//     buffer, so HBM streams while the current task iterates in registers;
//   * blur depth / sparse depth are read once with vectorised global loads, the result is written once;
//   * per iteration, x-neighbours come from warp shuffles, y-neighbours inside a thread from its own registers,
//     across warps from a double-buffered shared-memory row exchange, and across CTAs of the cluster from the same
//     exchange buffers written remotely through DSMEM with st.async, whose complete_tx lands on the consumer's
//     mbarrier: pure dataflow, one mbarrier wait per iteration and no cluster-wide barrier inside the loop.
// No tensor cores: a 9-point stencil with per-pixel weights is FMA-issue + HBM bound, not a contraction.
#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace cspn {

namespace {

constexpr int kMaxStrips = 128;
constexpr int kMaxBands = 64;
constexpr int kMaxPasses = 1024;
constexpr int kChainMaxIters = 32;    // chained strips: steps per pass whose recorded columns fit the history buffers

struct ClusterParams {
    const float* blur;    // [B*C][H][W]  d_0: the constant term always comes from here (cspn.py:58,76,81)
    const float* init;    // [B*C][H][W]  d at the start of this pass (null: d_0) -- passes after the first
    const float* sparse;  // [B][H][W] or null
    float* out;           // [B*C][H][W]
    float* iter_out;      // kStoreSteps / kAdjoint: where the result of this pass's FIRST step goes ([B*C][H][W] plane) ...
    long long iter_stride;  // ... and the (signed) distance in floats to the plane of the next step; the LAST step goes to `out`
    int C, H, W, gch, iters, norm_abs;
    int n_strips, n_bands, n_tasks;
    // fused final gather (cspn2d_fwd_gather_f32): the result is ALSO stored to these destinations -- the same block in
    // the gather buffers of the other GPUs (peer-mapped pointers over NVLink) and / or one NVLS multicast address that
    // the switch replicates to every GPU (multimem.st) -- tile by tile, while the kernel computes the next tiles
    float* out_peer[7];
    int n_peer;
    float* out_mc;
    unsigned long long* trace;   // -DCSPN_TRACE builds only (tools/trace_cluster.py): per-warp clock stamps, else null
    // chained strips (CHAIN kernels): the strips of an image are processed left to right; strip j records the column just left
    // of strip j+1 at every step (`hist`), so strip j+1 has an exact left neighbour and only its right edge goes stale
    float* hist;                 // [boundary block][step][warp][8] floats, block = (j * n_tasks / n_strips + q) * cluster size + CTA
    unsigned* flags;             // one word per block, zeroed before the launch; 1 = the block's history is complete
    int chain_lane;              // lane whose 4th column is recorded (the column left of the next strip's tile)
    int chain_group;             // image-channels per task group: tasks run group by group, strip-major inside a group, so that strip
                                 // j+1 of an image follows strip j by one group size: far enough for strip j to be finished, close
                                 // enough for the guidance columns the two tiles share to still be in L2 (the last group takes the rest)
    int tile_x0[kMaxStrips];  // column of the strip's first tile column (multiple of 4, may exceed image on the right)
    int ux0[kMaxStrips];      // useful (stored) columns [ux0, ux1)
    int ux1[kMaxStrips];
    int band_y0[kMaxBands];   // first row of the cluster's row range (one band unless the image is taller than a cluster)
    int uy0[kMaxBands];       // useful (stored) rows [uy0, uy1)
    int uy1[kMaxBands];
};

// ---- PTX helpers -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// lane-predicated forms: no divergent branch (BSSY/BSYNC) around the single arriving lane
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %1, 0;\n@p mbarrier.arrive.shared::cta.b64 _, [%0];\n}\n" ::"r"(bar), "r"((int)pred) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_if(uint32_t bar, uint32_t bytes, bool pred) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %2, 0;\n@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n}\n" ::"r"(bar), "r"(bytes), "r"((int)pred) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
// arrival that only signals progress (no memory ordering needed: it guards buffers this CTA has finished READING)
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_id_x() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_nclusterid_x() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
    return r;
}
// shared::cta address -> shared::cluster address of the same offset in CTA `rank`
__device__ __forceinline__ uint32_t map_to_cta(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
// remote store whose completion is signalled on the REMOTE mbarrier (complete_tx of the bytes stored)
__device__ __forceinline__ void st_async_v4(uint32_t remote_addr, float4 v, uint32_t remote_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(
                     remote_addr),
                 "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(remote_bar)
                 : "memory");
}
// 16-byte asynchronous copy global -> shared (LDGSTS): no register holds the data in flight
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// shared-memory accesses by 32-bit shared address (the chained-strip history: a generic pointer that varies per step makes
// ptxas rebuild the shared-window arithmetic at every access)
__device__ __forceinline__ float lds_f32(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ float4 lds_v4(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_v2(uint32_t a, float x, float y) { asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory"); }
__device__ __forceinline__ void sts_v4(uint32_t a, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// pull one box of a tensor into L2 (no shared-memory destination, no barrier): one instruction for a whole tile
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* map, int x, int y, int z) {
    asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(map), "r"(x), "r"(y), "r"(z) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int x, int y, int z, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
        "l"(map), "r"(x), "r"(y), "r"(z), "r"(bar)
        : "memory");
}

// ---- kernel ---------------------------------------------------------------------------------------
// Shared memory map (dynamic):
//   [0, 8*RB*TWP*4)           stage: 8 guidance planes [k][RB][TWP], TWP = TW + 8: the box of channel k starts at
//                             column tile_x0-4 (TMA needs a 16-byte aligned innermost origin, so the +-1 column
//                             shift of cspn.py:105-129 cannot ride on the box origin; the row shift dy_k does)
//   then xch[2][2*NW+2][TW]   row-exchange buffers (parity, slot, column)
//   then cbuf[RB][TW]         folded constant term c' of the current task
//   then 3 mbarriers          tma, full[0], full[1]
//
// Arithmetic is scalar FFMA: sm_90 has no packed FP32 FMA, and the stencil has no contraction for the tensor cores.
template <int PR, int PC, int NW>
struct Cfg {
    static constexpr int kThreads = 32 * NW;
    static constexpr int RB = NW * PR;   // rows per CTA band
    static constexpr int TW = 32 * PC;   // tile (strip) width
    static constexpr int TWP = TW + 8;   // staged row pitch: 4 apron columns on each side
    static constexpr int kSlots = 2 * NW + 2;
    // exchange rows carry 4 zero floats on each side: a thread reads the x-neighbours of a halo row straight from the
    // row (lane 0 / 31 find the zeros), so the halo taps need neither shuffles nor selects
    static constexpr int TWX = TW + 8;
    static constexpr size_t kPlaneBytes = (size_t)RB * TWP * sizeof(float);
    static constexpr size_t kStageBytes = 8 * kPlaneBytes;
    static constexpr size_t kXchParityBytes = (size_t)kSlots * TWX * sizeof(float);
    static constexpr size_t kXchBytes = 2 * kXchParityBytes;
    // the folded constant term c' (one float per pixel) lives in shared memory: it is read once per pixel and
    // iteration (one LDS.128 per patch row), which frees PR*PC registers per thread
    static constexpr size_t kCBytes = (size_t)RB * TW * sizeof(float);
    static constexpr size_t kSmemBytes = kStageBytes + kXchBytes + kCBytes + 64;
    // chained strips: the recorded column of the left neighbour strip (in) and of this strip (out), [step][warp][8 rows]
    static constexpr int kChainMaxIters = cspn::kChainMaxIters;
    static constexpr int kHistRow = NW * 8;
    static constexpr size_t kHistBytes = (size_t)kChainMaxIters * kHistRow * sizeof(float);
    static constexpr size_t kSmemBytesChain = kSmemBytes + 2 * kHistBytes;
    static constexpr bool kChainFits = kSmemBytesChain <= 232448 && PR <= 8;
    static_assert(PC == 4, "vectorised global/shared accesses below assume 4 columns per thread");
    static_assert(TWP <= 256, "TMA box <= 256 columns");
    static_assert(RB <= 256 && RB % 4 == 0, "TMA box rows; plane size must stay a multiple of 128 B");
    static_assert(PR >= 2, "a patch needs distinct top and bottom rows");
    static_assert(kSmemBytes <= 232448, "exceeds the 227 KB shared memory of an sm_90 CTA");
};

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.f32 %0, %1;" : "=f"(r) : "f"(x));   // 1/0 = inf, so 0 * (1/0) = NaN like the reference's 0/0; subnormal x: see exact_div
    return r;
}

// Extended row view: (-1) = left neighbour, (0..PC-1) = own pixels, (PC) = right neighbour.
template <int PC>
struct Row {
    const float (&v)[PC];
    const float (&ed)[2];
    __device__ __forceinline__ float operator()(int j) const { return j < 0 ? ed[0] : (j >= PC ? ed[1] : v[j]); }
};

// Channel of the tap that reads the pixel at offset (dy, dx) (channel order of cspn.py, see common.cuh):
//   (+1,+1)=0 (+1,0)=1 (+1,-1)=2 (0,+1)=3 (0,-1)=4 (-1,+1)=5 (-1,0)=6 (-1,-1)=7
__host__ __device__ constexpr int tap_of(int dy, int dx) { return dy == 1 ? 1 - dx : (dy == 0 ? (dx == 1 ? 3 : 4) : 6 - dx); }

__device__ __forceinline__ void load_row_smem(const float* p, float (&v)[4]) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void store_row_smem(float* p, const float (&v)[4]) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void store_row_remote(uint32_t addr, const float (&v)[4], uint32_t bar) {
    st_async_v4(addr, make_float4(v[0], v[1], v[2], v[3]), bar);
}

// -DCSPN_TRACE: clock stamps of cluster 0's tasks 1..kTraceTasks (steady state), lane 0 of every warp:
// trace[((slot*16 + cta)*8 + warp)*kTraceEvents + event].  Events: 0 task start, 1 guidance landed, 2 prologue done,
// 3 staging buffer released, 4 exchange buffers free, 5+3t / 6+3t / 7+3t = step t before wait / after wait / after
// publish, kTraceEvents-2 loop done, kTraceEvents-1 stored.
constexpr int kTraceTasks = 4, kTraceEvents = 5 + 3 * 64 + 2;
#ifdef CSPN_TRACE
#define CSPN_STAMP(xc, ev) do { if ((xc).tr) (xc).tr[(ev)] = clock64(); } while (0)
#else
#define CSPN_STAMP(xc, ev) do { } while (0)
#endif

// Per-thread constants of the row exchange.
struct Xch {
#ifdef CSPN_TRACE
    unsigned long long* tr;   // this warp's stamp row of the current task (lane 0, traced tasks only), else null
    int step;                 // running step index of the traced task
#endif
    float* base;          // xch + lane*PC (parity 0, slot 0)
    uint32_t bar_full0;   // local mbarriers: full[0], full[1] = full[0] + 8
    uint32_t rx_bytes;    // halo bytes this CTA receives per exchange
    // shared::cluster addresses in the neighbour CTAs (parity 0; parity 1 is a constant offset away)
    uint32_t up_data, up_bar;   // CTA above: its last slot ("halo from below") at my lane's columns, its full[0]
    uint32_t dn_data, dn_bar;   // CTA below: its slot 0 ("halo from above"), its full[0]
    bool has_up, has_dn;
    // warp roles as predicates for the branch-free publish: remote_up = this warp owns the CTA's top row and a CTA
    // above exists; remote_dn likewise
    bool remote_up, remote_dn;
    uint32_t my_tx;       // tx bytes this warp's lane-0 arrival arms: rx_bytes in the CTA's first warp, 0 elsewhere
    bool first_lane, last_lane;
    const float* cbuf;    // this thread's first pixel of c' (row r is r*TW floats further)
    // chained strips (CHAIN kernels; set per task)
    bool store_hist;      // this lane owns the recorded column and the strip has a right neighbour strip
    uint32_t hin;         // shared address of this warp's 8 floats of step 0 in the history-in buffer; history-out lies kHistBytes further
};

// Publish the boundary rows of the new d into exchange buffer PAR (local shared memory, and the neighbour CTAs'
// halo slots through DSMEM), then signal full[PAR].  Branch-free: roles are predicates.
template <int PR, int PC, int NW, int PAR>
__device__ __forceinline__ void publish(const Xch& x, int wy, const float (&top)[PC], const float (&bot)[PC]) {
    using K = Cfg<PR, PC, NW>;
    float* p = x.base + (size_t)PAR * K::kSlots * K::TWX;
    store_row_smem(p + (1 + 2 * wy) * K::TWX, top);
    store_row_smem(p + (2 + 2 * wy) * K::TWX, bot);
    const uint32_t bar = x.bar_full0 + 8 * PAR;
    // my top row is the "halo from below" (last slot) of the CTA above; my bottom row the "halo from above" below
    // (remote_up / remote_dn are warp-uniform by construction -- wy comes from a shuffle -- so these are uniform
    // branches, not divergence regions)
    if (x.remote_up) store_row_remote(x.up_data + PAR * (uint32_t)K::kXchParityBytes, top, x.up_bar + 8 * PAR);
    if (x.remote_dn) store_row_remote(x.dn_data + PAR * (uint32_t)K::kXchParityBytes, bot, x.dn_bar + 8 * PAR);
    __syncwarp();
    // one arrival per warp (lane 0); the first warp's also arms the bytes the neighbour CTAs will deliver (expect_tx of 0
    // bytes is a plain arrival): one predicated instruction and one predicate instead of two of each
    mbar_arrive_expect_tx_if(bar, x.my_tx, x.first_lane);
}

// ---- one propagation step ---------------------------------------------------------------------------------------
// d_it (din, with x-edges ein) -> d_{it+1} (dout, eout).  Reads exchange buffer PAR, publishes into PAR^1 (not on the last
// step).  Two register sets alternate as input and output: nothing is copied.
//
// What a neighbour waits for is my new boundary rows; what they wait for is the neighbours' previous boundary rows.  So
// after the mbarrier wait only the two halo rows remain to be added to the boundary rows: their x-neighbours are read
// from the padded exchange row itself (no shuffle, no select in the chain wait -> LDS -> 3 FMA -> STS) and the boundary
// rows are published at once.  ptxas schedules register arithmetic freely around the (volatile) barrier instructions and,
// left to itself, sinks most FMAs between the wait and the publish; memory operations however keep their order relative
// to the volatile asm statements, so the accumulators of the interior rows are seeded with c' (an LDS) only AFTER the
// publish: none of their 96 FMAs can run before it.  Per step: wait -> 24 halo FMAs -> publish -> [96 interior FMAs of
// this step, then the 40 own-row FMAs of the next step's boundary rows] -> wait.  On entry dout[0] and dout[PR-1] hold c'.
// Tile-edge lanes: the shuffled-in value of lane 0 (31) is meaningless; instead of zeroing it with a select per row and
// step, the three taps that would consume it are predicated off (exactly the reference's zero padding, NaN-safe).
// Measured alternatives (all own-row FMAs before the wait, wait forced late through a data dependency, source-major
// order over all interior rows, two phase-shifted warp groups) were no faster.
// scatter_row2: one source row into the accumulators of one destination row.  `src(jx)`, jx = -1..PC, is the extended
// source row; it sits SRC_DY rows below the destination row whose weights are `w`.  The loop nest is SOURCE-major: the FMAs
// that consume one source value are adjacent and write different accumulators (operand-reuse cache, no dependent pairs).
template <int PC, int SRC_DY, bool GUARD, typename Src>
__device__ __forceinline__ void scatter_row2(const float (&w)[PC][8], const Src& src, float (&acc)[PC], bool use_left,
                                             bool use_right) {
#pragma unroll
    for (int jx = 0; jx <= PC + 1; ++jx) {
        const int sx = jx <= PC - 1 ? jx : (jx == PC ? -1 : PC);   // own columns first, then the left / right neighbour
        const float xv = src(sx);
#pragma unroll
        for (int dx = 1; dx >= -1; --dx) {
            const int j = sx - dx;
            if (j < 0 || j >= PC) continue;
            if (SRC_DY == 0 && dx == 0) continue;
            if (GUARD && sx < 0) { if (use_left) acc[j] = fmaf(w[j][tap_of(SRC_DY, dx)], xv, acc[j]); }
            else if (GUARD && sx >= PC) { if (use_right) acc[j] = fmaf(w[j][tap_of(SRC_DY, dx)], xv, acc[j]); }
            else acc[j] = fmaf(w[j][tap_of(SRC_DY, dx)], xv, acc[j]);
        }
    }
}
template <int PC>
__device__ __forceinline__ void row_edges_raw(const float (&v)[PC], float (&ed)[2]) {
    ed[0] = __shfl_up_sync(0xffffffffu, v[PC - 1], 1);     // lane 0 gets its own value back: never consumed (guarded taps)
    ed[1] = __shfl_down_sync(0xffffffffu, v[0], 1);
}

// CHAIN (chained strips).  A history row holds, for one step t and one warp, the recorded column at time t: [0..3] the warp's
// rows 0..3, [4] the row above its patch, [5] the row below, [6] its row 4.  `hrow` = this warp's slot of row t of the step
// being taken.  The lane that owns the recorded column stores row t after the wait (it then holds all seven values: its
// input rows and the two halo rows); lane 0 reads its halo rows' column -1 from row t instead of the zero pad (a pointer
// select: no extra load) and, at the end of the step, the column -1 of its own rows for the next step from row t+1.  A strip
// without a left neighbour reads a zero-filled history: the reference's zero padding, so the left taps of lane 0 are never
// predicated off in these kernels.
template <int PR, int PC, int NW, int PAR, bool PUBLISH, bool CHAIN = false>
__device__ __forceinline__ void iterate3(const Xch& x, int wy, uint32_t phase, const float (&w)[PR][PC][8],
                                         float (&din)[PR][PC], const float (&ein)[PR][2], float (&dout)[PR][PC],
                                         float (&eout)[PR][2], uint32_t hrow = 0) {
    using K = Cfg<PR, PC, NW>;
    const bool ul = CHAIN ? true : !x.first_lane, ur = !x.last_lane;
    // ---- A: own-row taps of the two boundary rows ----------------------------------------------------------------
    scatter_row2<PC, 0, true>(w[0], Row<PC>{din[0], ein[0]}, dout[0], ul, ur);
    scatter_row2<PC, +1, true>(w[0], Row<PC>{din[1], ein[1]}, dout[0], ul, ur);
    scatter_row2<PC, 0, true>(w[PR - 1], Row<PC>{din[PR - 1], ein[PR - 1]}, dout[PR - 1], ul, ur);
    scatter_row2<PC, -1, true>(w[PR - 1], Row<PC>{din[PR - 2], ein[PR - 2]}, dout[PR - 1], ul, ur);
    // ---- B: the neighbours' rows, then publish at once ---------------------------------------------------------------
#ifndef CSPN_ABLATE_NO_SYNC
    CSPN_STAMP(x, 5 + 3 * x.step);
    mbar_wait(x.bar_full0 + 8 * PAR, phase);
    CSPN_STAMP(x, 6 + 3 * x.step);
#endif
    {
        const float* p = x.base + (size_t)PAR * K::kSlots * K::TWX;
        const float* pu = p + (2 * wy) * K::TWX;          // row above my patch
        const float* pd = p + (2 * wy + 3) * K::TWX;      // row below my patch
        float u[PC], ue[2], d[PC], de[2];
        load_row_smem(pu, u);
        load_row_smem(pd, d);
        if constexpr (CHAIN) {
            ue[0] = lds_f32(x.first_lane ? hrow + 16 : smem_u32(pu - 1));
            de[0] = lds_f32(x.first_lane ? hrow + 20 : smem_u32(pd - 1));
            if (x.store_hist) {
                const uint32_t q = hrow + (uint32_t)K::kHistBytes;      // history-out
                sts_v4(q, make_float4(din[0][PC - 1], din[1][PC - 1], din[PR > 2 ? 2 : 0][PC - 1], din[PR > 3 ? 3 : 0][PC - 1]));
                sts_v2(q + 16, u[PC - 1], d[PC - 1]);
                if constexpr (PR > 4) sts_f32(q + 24, din[PR > 4 ? 4 : 0][PC - 1]);
            }
        } else {
            ue[0] = pu[-1];                               // pad floats are zero at the tile edges
            de[0] = pd[-1];
        }
        ue[1] = pu[PC];
        de[1] = pd[PC];
        scatter_row2<PC, -1, false>(w[0], Row<PC>{u, ue}, dout[0], true, true);
        scatter_row2<PC, +1, false>(w[PR - 1], Row<PC>{d, de}, dout[PR - 1], true, true);
    }
    if constexpr (PUBLISH) {
#ifndef CSPN_ABLATE_NO_SYNC
        publish<PR, PC, NW, PAR ^ 1>(x, wy, dout[0], dout[PR - 1]);
        CSPN_STAMP(x, 7 + 3 * x.step);
#else
        asm volatile("" ::: "memory");
#endif
        row_edges_raw<PC>(dout[0], eout[0]);
        row_edges_raw<PC>(dout[PR - 1], eout[PR - 1]);
    }
    // ---- C: interior rows (their seed is loaded after the publish: see above) ---------------------------------------------
#if defined(CSPN_STEP_SRCMAJOR)
    // experiment: source-major over ALL interior destination rows: the (up to 8) FMAs that consume one source value adjacent
#pragma unroll
    for (int r = 1; r + 1 < PR; ++r) load_row_smem(x.cbuf + r * K::TW, dout[r]);
#pragma unroll
    for (int sr = 0; sr < PR; ++sr) {
        const Row<PC> src{din[sr], ein[sr]};
#pragma unroll
        for (int jx = 0; jx <= PC + 1; ++jx) {
            const int sx = jx <= PC - 1 ? jx : (jx == PC ? -1 : PC);
            const float xv = src(sx);
#pragma unroll
            for (int dy = 1; dy >= -1; --dy) {       // source row sr lies dy rows below destination row sr - dy
                const int r = sr - dy;
                if (r < 1 || r > PR - 2) continue;
#pragma unroll
                for (int dx = 1; dx >= -1; --dx) {
                    const int j = sx - dx;
                    if (j < 0 || j >= PC) continue;
                    if (dy == 0 && dx == 0) continue;
                    if (sx < 0) { if (ul) dout[r][j] = fmaf(w[r][j][tap_of(dy, dx)], xv, dout[r][j]); }
                    else if (sx >= PC) { if (ur) dout[r][j] = fmaf(w[r][j][tap_of(dy, dx)], xv, dout[r][j]); }
                    else dout[r][j] = fmaf(w[r][j][tap_of(dy, dx)], xv, dout[r][j]);
                }
            }
        }
    }
    if constexpr (PUBLISH) {
#pragma unroll
        for (int r = 1; r + 1 < PR; ++r) row_edges_raw<PC>(dout[r], eout[r]);
    }
#else
#pragma unroll
    for (int r = 1; r + 1 < PR; ++r) {
        load_row_smem(x.cbuf + r * K::TW, dout[r]);
        scatter_row2<PC, -1, true>(w[r], Row<PC>{din[r - 1], ein[r - 1]}, dout[r], ul, ur);
        scatter_row2<PC, 0, true>(w[r], Row<PC>{din[r], ein[r]}, dout[r], ul, ur);
        scatter_row2<PC, +1, true>(w[r], Row<PC>{din[r + 1], ein[r + 1]}, dout[r], ul, ur);
        if constexpr (PUBLISH) row_edges_raw<PC>(dout[r], eout[r]);
    }
#endif
    if constexpr (CHAIN && PUBLISH) {   // column -1 of my rows at the next step (row t+1 of the history)
        const uint32_t hn = hrow + K::kHistRow * 4;
        const float4 h = lds_v4(hn);
        eout[0][0] = x.first_lane ? h.x : eout[0][0];
        eout[1][0] = x.first_lane ? h.y : eout[1][0];
        if constexpr (PR > 2) eout[2][0] = x.first_lane ? h.z : eout[2][0];
        if constexpr (PR > 3) eout[3][0] = x.first_lane ? h.w : eout[3][0];
        if constexpr (PR > 4) eout[4][0] = x.first_lane ? lds_f32(hn + 24) : eout[4][0];
        static_assert(PR <= 5, "a history row has room for five patch rows");
    }
    if constexpr (PUBLISH) {   // seeds of the next step's boundary rows, into the now dead input set
        load_row_smem(x.cbuf, din[0]);
        load_row_smem(x.cbuf + (PR - 1) * K::TW, din[PR - 1]);
    }
}

template <int PR, int PC, int NW, int PAR, bool PUBLISH, bool CHAIN = false>
__device__ __forceinline__ void step_fwd(Xch& x, int wy, uint32_t phase, const float (&w)[PR][PC][8],
                                         float (&din)[PR][PC], float (&ein)[PR][2], float (&dout)[PR][PC],
                                         float (&eout)[PR][2], uint32_t hrow = 0) {
    iterate3<PR, PC, NW, PAR, PUBLISH, CHAIN>(x, wy, phase, w, din, ein, dout, eout, hrow);
#ifdef CSPN_TRACE
    ++x.step;
#endif
}

// What a launch computes with the folded weights w' it builds in its prologue:
//   kForward     d <- c' + sum_k w'_k shift_k(d), `iters` times                                   (the product path)
//   kStoreSteps  the same, and every step's result is also written to global memory (the forward iterates d_1..d_N
//                that the backward pass needs)
//   kAdjoint     lambda <- sum_k shift_{-k}(w'_k lambda), `iters` times, every step's result written out: the
//                transpose of the forward step (cspn2d_bwd.cu has the derivation); `blur` carries lambda's start value
enum ClusterMode { kForward = 0, kStoreSteps = 1, kAdjoint = 2 };

// Adjoint of scatter_row: the SOURCE pixels (weights w, values l) of one row push w_k * l into the destination row DY
// rows further down (off_k = (DY, dx)): destination column = source column + dx.  Columns -1 and PC belong to the
// neighbouring lanes and are collected in xl / xr.
template <int PC, int DY>
__device__ __forceinline__ void adj_row(const float (&w)[PC][8], const float (&l)[PC], float (&acc)[PC], float& xl, float& xr) {
#pragma unroll
    for (int j = 0; j < PC; ++j) {
#pragma unroll
        for (int dx = 1; dx >= -1; --dx) {
            if (DY == 0 && dx == 0) continue;
            const int jd = j + dx;
            const float wk = w[j][tap_of(DY, dx)];
            if (jd < 0) xl = fmaf(wk, l[j], xl);
            else if (jd >= PC) xr = fmaf(wk, l[j], xr);
            else acc[jd] = fmaf(wk, l[j], acc[jd]);
        }
    }
}
// hand the out-of-thread columns to the neighbouring lanes: my xr is lane+1's column 0, my xl is lane-1's column PC-1
template <int PC>
__device__ __forceinline__ void fold_edges(float (&v)[PC], float xl, float xr, bool first_lane, bool last_lane) {
    const float from_left = __shfl_up_sync(0xffffffffu, xr, 1);
    const float from_right = __shfl_down_sync(0xffffffffu, xl, 1);
    v[0] += first_lane ? 0.f : from_left;
    v[PC - 1] += last_lane ? 0.f : from_right;
}

// One adjoint step lin = lambda_{t+1} -> lout = lambda_t.  The partial rows owed to the warps above / below depend on
// lin only, so they are published FIRST (exchange buffer PAR) and the wait for the neighbours' rows comes last.
template <int PR, int PC, int NW, int PAR>
__device__ __forceinline__ void iterate_adj(const Xch& x, int wy, uint32_t phase, const float (&w)[PR][PC][8],
                                            const float (&lin)[PR][PC], float (&lout)[PR][PC]) {
    using K = Cfg<PR, PC, NW>;
    {
        float up[PC], dn[PC], upl = 0.f, upr = 0.f, dnl = 0.f, dnr = 0.f;
#pragma unroll
        for (int j = 0; j < PC; ++j) { up[j] = 0.f; dn[j] = 0.f; }
        adj_row<PC, -1>(w[0], lin[0], up, upl, upr);             // my top row feeds the row above my patch
        adj_row<PC, +1>(w[PR - 1], lin[PR - 1], dn, dnl, dnr);   // my bottom row feeds the row below
        fold_edges<PC>(up, upl, upr, x.first_lane, x.last_lane);
        fold_edges<PC>(dn, dnl, dnr, x.first_lane, x.last_lane);
        publish<PR, PC, NW, PAR>(x, wy, up, dn);
    }
    float xl[PR], xr[PR];
#pragma unroll
    for (int r = 0; r < PR; ++r) {
        xl[r] = 0.f; xr[r] = 0.f;
#pragma unroll
        for (int j = 0; j < PC; ++j) lout[r][j] = 0.f;
    }
#pragma unroll
    for (int r = 0; r < PR; ++r) {                               // source rows
        if (r > 0) adj_row<PC, -1>(w[r], lin[r], lout[r - 1], xl[r - 1], xr[r - 1]);
        adj_row<PC, 0>(w[r], lin[r], lout[r], xl[r], xr[r]);
        if (r + 1 < PR) adj_row<PC, +1>(w[r], lin[r], lout[r + 1], xl[r + 1], xr[r + 1]);
    }
#pragma unroll
    for (int r = 0; r < PR; ++r) fold_edges<PC>(lout[r], xl[r], xr[r], x.first_lane, x.last_lane);
    mbar_wait(x.bar_full0 + 8 * PAR, phase);
    {
        const float* p = x.base + (size_t)PAR * K::kSlots * K::TWX;
        float a[PC], b[PC];
        load_row_smem(p + (2 * wy) * K::TWX, a);        // what the warp above owes my top row
        load_row_smem(p + (2 * wy + 3) * K::TWX, b);    // what the warp below owes my bottom row
#pragma unroll
        for (int j = 0; j < PC; ++j) { lout[0][j] += a[j]; lout[PR - 1][j] += b[j]; }
    }
}

// GENERAL = false compiles out row bands and the continuation input of multi-pass plans: the common single-pass,
// single-band launch (every BASELINE 2D config) pays nothing for them.
template <int PR, int PC, int NW, bool ABS, bool GENERAL, int MODE = kForward, bool CHAIN = false>
__global__ void __launch_bounds__(32 * NW, 1)
cspn2d_cluster_kernel(const __grid_constant__ CUtensorMap tm_guidance, const __grid_constant__ CUtensorMap tm_blur,
                      const __grid_constant__ CUtensorMap tm_sparse, const __grid_constant__ ClusterParams prm) {
    using K = Cfg<PR, PC, NW>;
    constexpr int RB = K::RB, TW = K::TW, TWP = K::TWP, TWX = K::TWX;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* stage = reinterpret_cast<float*>(smem_raw);
    float* xch = reinterpret_cast<float*>(smem_raw + K::kStageBytes);
    float* cbuf = reinterpret_cast<float*>(smem_raw + K::kStageBytes + K::kXchBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + K::kStageBytes + K::kXchBytes + K::kCBytes);
    const uint32_t bar_tma = smem_u32(bars), bar_full0 = smem_u32(bars + 1);
    [[maybe_unused]] float* hist_in = reinterpret_cast<float*>(smem_raw + K::kSmemBytes);   // CHAIN: [step][warp][8], then history-out
    static_assert(!CHAIN || (MODE == kForward && K::kChainFits), "chained strips: forward kernels of the 8-warp configurations");

    const int tid = threadIdx.x, lane = tid & 31;
    const int wy = __shfl_sync(0xffffffffu, tid >> 5, 0);   // warp index, provably warp-uniform for the compiler
    const uint32_t crank = cluster_ctarank(), csize = cluster_nctarank();
    const int H = prm.H, W = prm.W;
    const int cta_dy = (int)crank * RB;     // first row of this CTA / of this thread, relative to the task's band origin
    const int thr_dy = cta_dy + wy * PR;
    const size_t HW = (size_t)H * W;

    Xch xc;
#ifdef CSPN_TRACE
    xc.tr = nullptr;
    xc.step = 0;
#endif
    xc.base = xch + 4 + lane * PC;     // 4 zero floats lead every exchange row
    xc.bar_full0 = bar_full0;
    xc.has_up = crank > 0;
    xc.has_dn = crank + 1 < csize;
    xc.up_data = xc.has_up ? map_to_cta(smem_u32(xc.base + (K::kSlots - 1) * TWX), crank - 1) : 0u;
    xc.up_bar = xc.has_up ? map_to_cta(bar_full0, crank - 1) : 0u;
    xc.dn_data = xc.has_dn ? map_to_cta(smem_u32(xc.base), crank + 1) : 0u;
    xc.dn_bar = xc.has_dn ? map_to_cta(bar_full0, crank + 1) : 0u;
    xc.rx_bytes = (uint32_t)((xc.has_up ? 1 : 0) + (xc.has_dn ? 1 : 0)) * TW * sizeof(float);
    xc.remote_up = xc.has_up && wy == 0;
    xc.remote_dn = xc.has_dn && wy == NW - 1;
    xc.my_tx = wy == 0 ? xc.rx_bytes : 0u;
    xc.first_lane = lane == 0;
    xc.last_lane = lane == 31;
    xc.cbuf = cbuf + (size_t)(wy * PR) * TW + lane * PC;
    xc.store_hist = false; xc.hin = 0;
    if constexpr (CHAIN) xc.hin = smem_u32(hist_in + wy * 8);

    // Persistent clusters: cluster q runs tasks q, q + Q, q + 2Q, ...  (task = (image*C + channel, strip))
    const int n_tasks = prm.n_tasks;
    const int task_stride = (int)cluster_nclusterid_x();
    int task = (int)cluster_id_x();

    // Stage the 8 guidance planes of one task: rows shifted by dy_k ride on the box origin; out-of-image rows and
    // columns arrive as zeros (= ZeroPad2d, cspn.py:105-129).
    // CHAIN task order: groups of prm.chain_group image-channels, strip-major inside a group
    [[maybe_unused]] auto chain_decode = [&](int t, int& strip_o, int& q_o) {
        const int nq_all = prm.n_tasks / prm.n_strips, g = prm.chain_group;
        const int per_group = g * prm.n_strips;
        int grp = t / per_group;
        const int n_groups = nq_all / g;                 // >= 1; the last group also holds the remainder
        if (grp >= n_groups) grp = n_groups - 1;
        const int t2 = t - grp * per_group;
        const int size = (grp == n_groups - 1) ? nq_all - grp * g : g;
        strip_o = t2 / size;
        q_o = grp * g + t2 % size;
    };
    auto issue_stage = [&](int t) {
        // task order: strips of one image are neighbours (default), or strip-major when the strips are chained (a task's
        // left neighbour strip is then n_tasks / n_strips tasks back: finished long before, whatever cluster ran it)
        int strip_t = t % prm.n_strips, q_t = t / prm.n_strips;
        if constexpr (CHAIN) chain_decode(t, strip_t, q_t);
        const int band_t = GENERAL ? q_t % prm.n_bands : 0;
        const int b_t = (GENERAL ? q_t / prm.n_bands : q_t) / prm.C;
        mbar_arrive_expect_tx(bar_tma, (uint32_t)K::kStageBytes);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            tma_load_3d(smem_u32(stage) + (uint32_t)(k * K::kPlaneBytes), &tm_guidance, prm.tile_x0[strip_t] - 4,
                        (GENERAL ? prm.band_y0[band_t] : 0) + cta_dy + off2_dy(k), b_t * prm.gch + k, bar_tma);
    };

    if (tid == 0) {
        mbar_init(bar_tma, 1);
        mbar_init(bar_full0, NW);
        mbar_init(bar_full0 + 8, NW);
        fence_barrier_init();
        fence_proxy_async();
        if (task < n_tasks) issue_stage(task);
    }
    // every CTA's barriers must be initialised before a neighbour's st.async can target them
    cluster_arrive();
    // halo slots without a neighbour stay zero for the whole kernel (rows outside the image), and so do the 4 pad
    // floats on either side of every row (columns outside the tile).  Nobody else ever writes these locations.
    if (!xc.has_up)
        for (int i = tid; i < TWX; i += K::kThreads) { xch[i] = 0.f; xch[(size_t)K::kSlots * TWX + i] = 0.f; }
    if (!xc.has_dn)
        for (int i = tid; i < TWX; i += K::kThreads) {
            xch[(size_t)(K::kSlots - 1) * TWX + i] = 0.f;
            xch[(size_t)(2 * K::kSlots - 1) * TWX + i] = 0.f;
        }
    for (int i = tid; i < 2 * K::kSlots * 8; i += K::kThreads) {
        const int row = i >> 3, c = i & 7;
        xch[(size_t)row * TWX + (c < 4 ? c : TW + c)] = 0.f;
    }
    cluster_wait();

    uint32_t ph_tma = 0, ph0 = 0, ph1 = 0;  // phase parities of the three mbarriers (they run on across tasks)
    bool first = true;
    for (; task < n_tasks; task += task_stride) {
        const int nq = prm.n_tasks / prm.n_strips;
        int strip = task % prm.n_strips, qi = task / prm.n_strips;      // qi: image-channel (x band)
        if constexpr (CHAIN) chain_decode(task, strip, qi);
        const int band = GENERAL ? qi % prm.n_bands : 0;
        const int bc = GENERAL ? qi / prm.n_bands : qi;  // b*C + c
        const int b = bc / prm.C;
        const int y_thr = (GENERAL ? prm.band_y0[band] : 0) + thr_dy;   // first image row of this thread
        const float* init = GENERAL ? prm.init : nullptr;
        const int tile_x0 = prm.tile_x0[strip];
        const int x_thr = tile_x0 + lane * PC;  // first column of this thread
#ifdef CSPN_TRACE
        {
            const int slot = (task - (int)cluster_id_x()) / task_stride - 1;    // the cluster's 2nd, 3rd, ... task
            xc.tr = (prm.trace && cluster_id_x() == 0 && lane == 0 && slot >= 0 && slot < kTraceTasks)
                        ? prm.trace + ((size_t)(slot * 16 + (int)crank) * 8 + wy) * kTraceEvents : nullptr;
            xc.step = 0;
        }
        CSPN_STAMP(xc, 0);
#endif

        // chained strip with a left neighbour: ask for that strip's "history complete" flag now, look at the answer after the
        // loads below have been issued (it was set long ago unless the batch is small)
        [[maybe_unused]] unsigned hist_ready = 1u;
        [[maybe_unused]] const unsigned* hist_flag = nullptr;
        if constexpr (CHAIN) {
            if (strip > 0) {
                hist_flag = prm.flags + ((size_t)(strip - 1) * nq + qi) * csize + crank;
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(hist_ready) : "l"(hist_flag) : "memory");
            }
        }

        // ---- thread state ---------------------------------------------------------------------------
        float w[PR][PC][8], d[PR][PC];
        const float* blur = prm.blur + (size_t)bc * HW;
        const float* sparse = prm.sparse ? prm.sparse + (size_t)b * HW : nullptr;

        // blur_depth rows go global -> shared with cp.async, straight into this thread's slots of the c' buffer (free until
        // the prologue writes c' there): nothing holds them in flight, and the prologue reads each row back when it needs
        // it.  sparse_depth rows (only their sign is used) wait in registers and are converted row by row.  Both were
        // pulled into L2 one task ago by the TMA prefetch below, so what is hidden here is an L2 latency.
        // W % 4 == 0 and x_thr % 4 == 0: a float4 is entirely inside or outside the image.
        const bool col_in = (x_thr >= 0) && (x_thr < W);
        float4 sv[PR];
        float* my_c = const_cast<float*>(xc.cbuf);
#pragma unroll
        for (int r = 0; r < PR; ++r) {
            const int y = y_thr + r;
            sv[r] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (col_in && y < H) {
                cp_async16(smem_u32(my_c + r * TW), blur + (size_t)y * W + x_thr);
                if (sparse) sv[r] = __ldg(reinterpret_cast<const float4*>(sparse + (size_t)y * W + x_thr));
            } else {
                *reinterpret_cast<float4*>(my_c + r * TW) = sv[r];       // outside the image: d = 0
            }
        }
        // the neighbours have finished reading the exchange buffers of the previous task (they arrived right after their
        // step loop): waited for here, under the loads
        if (!first) cluster_wait();
        [[maybe_unused]] bool has_out = false;
        if constexpr (CHAIN) {
            const bool has_in = strip > 0;
            has_out = strip + 1 < prm.n_strips;
            xc.store_hist = has_out && lane == prm.chain_lane;
            if (!has_in) {      // image border on the left: column -1 is the reference's zero padding
                const int n16 = prm.iters * K::kHistRow / 4;
                for (int i = tid; i < n16; i += K::kThreads) reinterpret_cast<float4*>(hist_in)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            } else {
                // the left neighbour strip's history block of this CTA's rows must be complete (normally it has been for a
                // long time); then pull it into shared memory: it is first read after the prologue's barrier
                const size_t blk = ((size_t)(strip - 1) * nq + qi) * csize + crank;
                while (hist_ready == 0u)
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(hist_ready) : "l"(hist_flag) : "memory");
                const int n16 = prm.iters * K::kHistRow / 4;
                const float* src = prm.hist + blk * (size_t)(prm.iters * K::kHistRow);
                for (int i = tid; i < n16; i += K::kThreads) cp_async16(smem_u32(hist_in + 4 * i), src + 4 * i);
            }
        }
        // the first row exchange of a task needs only blur_depth: it is published from inside the prologue (after row 0),
        // so its DSMEM round trip hides under the normalisation of the other rows instead of stalling the first step.
        // (A continuation pass starts from the previous pass's result, read further down: it publishes after the prologue.)
        const bool early_publish = (MODE != kAdjoint) && !(GENERAL && init != nullptr);

        mbar_wait(bar_tma, ph_tma);
        ph_tma ^= 1;
        CSPN_STAMP(xc, 1);

        // ---- prologue: affinity normalisation + mask folding (cspn.py:85-144, 63-64) ------------------
        // a_k(y,x) = g_k(y+dy_k, x+dx_k): dy_k came with the TMA box, dx_k is applied here: the thread reads its own
        // PC columns of plane k and takes the missing neighbour column from the next / previous lane (tile edge
        // lanes read the apron column of the staged row instead).
#pragma unroll
        for (int r = 0; r < PR; ++r) {
            const int y = y_thr + r;
            float S[PC], A[PC], a[8][PC];
#pragma unroll
            for (int j = 0; j < PC; ++j) { S[j] = 0.f; A[j] = 0.f; }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float* row = stage + ((size_t)k * RB + wy * PR + r) * TWP + 4 + lane * PC;
                float v[PC];
                load_row_smem(row, v);
                if (off2_dx(k) == 1) {
                    float nb = __shfl_down_sync(0xffffffffu, v[0], 1);
                    if (lane == 31) nb = row[PC];
#pragma unroll
                    for (int j = 0; j < PC - 1; ++j) a[k][j] = v[j + 1];
                    a[k][PC - 1] = nb;
                } else if (off2_dx(k) == -1) {
                    float nb = __shfl_up_sync(0xffffffffu, v[PC - 1], 1);
                    if (lane == 0) nb = row[-1];
#pragma unroll
                    for (int j = PC - 1; j > 0; --j) a[k][j] = v[j - 1];
                    a[k][0] = nb;
                } else {
#pragma unroll
                    for (int j = 0; j < PC; ++j) a[k][j] = v[j];
                }
#pragma unroll
                for (int j = 0; j < PC; ++j) {
                    if (ABS) a[k][j] = fabsf(a[k][j]);        // cspn.py:88-89
                    S[j] += fabsf(a[k][j]);                    // cspn.py:135-136
                    A[j] += a[k][j];                           // numerator of gate_sum, cspn.py:139
                }
            }
            // this row's blur_depth (from the c' slot the cp.async filled) and mask
            if (r == 0) cp_async_wait_all();            // this thread's own copies: no barrier needed
            load_row_smem(my_c + r * TW, d[r]);
            const float mrow[PC] = {signf(sv[r].x), signf(sv[r].y), signf(sv[r].z), signf(sv[r].w)};
            if (r == 0 && early_publish) {
                float bot[PC];
                load_row_smem(my_c + (PR - 1) * TW, bot);
                publish<PR, PC, NW, 0>(xc, wy, d[0], bot);
            }
            float cj[PC];
            bool exact_div = false;
#pragma unroll
            for (int j = 0; j < PC; ++j) {
                const bool in = col_in && (y < H);
                const float inv = rcp_approx(S[j]);
                const float om = 1.f - mrow[j];
                const float scale = in ? om * inv : 0.f;      // pixels outside the image: w = 0, c = 0, d = 0 forever
                float sw = 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k) { w[r][j][k] = a[k][j] * scale; sw += w[r][j][k]; }
                // (1-m)(1 - gate_sum) + m == 1 - sum_k w'_k, formed from the quotients as cspn.py:139 does
                cj[j] = in ? (1.f - sw) * d[r][j] : 0.f;
                // a * (1/S) is a / S to 2 ulp and has the same 0/0, x/inf and inf/inf results, EXCEPT when 1/S overflows
                // (S subnormal): there the reference's quotient (cspn.py:138) is an ordinary number
                exact_div |= in && (inv > 8.0e37f);
            }
            if (exact_div) {                                   // cold: IEEE division, the reference's own expression
#pragma unroll
                for (int j = 0; j < PC; ++j) {
                    const float om = 1.f - mrow[j];
                    float gsum = 0.f;
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float q = __fdiv_rn(a[k][j], S[j]);
                        gsum += q;                             // gate_sum, cspn.py:139
                        w[r][j][k] = om * q;
                    }
                    cj[j] = (om * (1.f - gsum) + mrow[j]) * d[r][j];
                }
            }
            // only this thread ever reads these values back: no barrier needed
            if constexpr (MODE != kAdjoint) {
                store_row_smem(const_cast<float*>(xc.cbuf) + r * TW, cj);   // the adjoint has no constant term
            }
            // a pass after the first continues from the previous pass's result; c' above still used d_0
            if (GENERAL && init != nullptr && col_in && y < H) {
                const float4 iv = __ldg(reinterpret_cast<const float4*>(init + (size_t)bc * HW + (size_t)y * W + x_thr));
                d[r][0] = iv.x; d[r][1] = iv.y; d[r][2] = iv.z; d[r][3] = iv.w;
            }
        }
        CSPN_STAMP(xc, 2);
        __syncthreads();  // every warp is done with the staging buffer
        CSPN_STAMP(xc, 3);

        // ---- next task's guidance starts streaming in now; it lands while this task iterates in registers ----
        const int next = task + task_stride;
        if (next < n_tasks) {
            if (tid == 0) {
                fence_proxy_async();  // generic-proxy reads of `stage` above are ordered before the async-proxy writes
                issue_stage(next);
                // its blur / sparse rows: one TMA prefetch each pulls the CTA's whole tile into L2 (two instructions per CTA
                // and task; the per-thread prefetch loop this replaces cost 1 250 cycles of every task)
                int strip_n = next % prm.n_strips, q_n = next / prm.n_strips;
                if constexpr (CHAIN) chain_decode(next, strip_n, q_n);
                const int bc_n = GENERAL ? q_n / prm.n_bands : q_n;
                const int y_n = (GENERAL ? prm.band_y0[q_n % prm.n_bands] : 0) + cta_dy;
                tma_prefetch_3d(&tm_blur, prm.tile_x0[strip_n], y_n, bc_n);
                if (prm.sparse) tma_prefetch_3d(&tm_sparse, prm.tile_x0[strip_n], y_n, bc_n / prm.C);
            }
        }

        // ---- the N iterations: registers only, one mbarrier wait each ----------------------------------
        first = false;
        CSPN_STAMP(xc, 4);
        const int iters = prm.iters;
        // kStoreSteps / kAdjoint: every step's result also goes to global memory (useful pixels only); the pass's last
        // step leaves through the epilogue
        [[maybe_unused]] float* step_ptr = nullptr;
        [[maybe_unused]] unsigned step_rows = 0;      // bit r: row r of this thread is stored
        if constexpr (MODE != kForward) {
            const int sy0 = GENERAL ? prm.uy0[band] : 0, sy1 = GENERAL ? prm.uy1[band] : H;
            if (x_thr >= prm.ux0[strip] && x_thr < prm.ux1[strip]) {
#pragma unroll
                for (int r = 0; r < PR; ++r)
                    if (y_thr + r >= sy0 && y_thr + r < sy1) step_rows |= 1u << r;
            }
            step_ptr = prm.iter_out + (size_t)bc * HW + (size_t)y_thr * W + x_thr;
        }
        [[maybe_unused]] auto store_step = [&](const float (&v)[PR][PC]) {
#pragma unroll
            for (int r = 0; r < PR; ++r)
                if (step_rows & (1u << r))
                    *reinterpret_cast<float4*>(step_ptr + (size_t)r * W) = make_float4(v[r][0], v[r][1], v[r][2], v[r][3]);
            step_ptr += prm.iter_stride;
        };
        if constexpr (MODE == kAdjoint) {
            float d2[PR][PC];               // (d -> d2) on even steps, back on odd ones
            int it = 0;
            for (; it + 2 <= iters; it += 2) {
                iterate_adj<PR, PC, NW, 0>(xc, wy, ph0, w, d, d2);
                ph0 ^= 1;
                store_step(d2);
                iterate_adj<PR, PC, NW, 1>(xc, wy, ph1, w, d2, d);
                ph1 ^= 1;
                if (it + 2 < iters) store_step(d);
            }
            if (it < iters) {
                iterate_adj<PR, PC, NW, 0>(xc, wy, ph0, w, d, d2);
                ph0 ^= 1;
#pragma unroll
                for (int r = 0; r < PR; ++r)
#pragma unroll
                    for (int j = 0; j < PC; ++j) d[r][j] = d2[r][j];
            }
            cluster_arrive_relaxed();
        } else {
#ifndef CSPN_ABLATE_NO_SYNC
        if (!early_publish) publish<PR, PC, NW, 0>(xc, wy, d[0], d[PR - 1]);
#endif
        float e[PR][2];                 // x-edges (left, right neighbour) of the rows of d
#pragma unroll
        for (int r = 0; r < PR; ++r) row_edges_raw<PC>(d[r], e[r]);
        if constexpr (CHAIN) {          // column -1 of lane 0's rows at step 0 (row 0 of the history)
#pragma unroll
            for (int r = 0; r < PR; ++r) e[r][0] = xc.first_lane ? lds_f32(xc.hin + 4 * (r < 4 ? r : 6)) : e[r][0];
        }
        float d2[PR][PC], e2[PR][2];    // second register set: (d,e) -> (d2,e2) on even steps, back on odd ones
#pragma unroll
        for (int r = 0; r < PR; ++r) load_row_smem(xc.cbuf + r * TW, d2[r]);   // accumulators of the first step start from c'
        int it = 0;
        for (; it + 2 < iters; it += 2) {   // steady state: every step publishes
            step_fwd<PR, PC, NW, 0, true, CHAIN>(xc, wy, ph0, w, d, e, d2, e2, xc.hin + it * (K::kHistRow * 4));
            ph0 ^= 1;
            if constexpr (MODE == kStoreSteps) store_step(d2);
            step_fwd<PR, PC, NW, 1, true, CHAIN>(xc, wy, ph1, w, d2, e2, d, e, xc.hin + (it + 1) * (K::kHistRow * 4));
            ph1 ^= 1;
            if constexpr (MODE == kStoreSteps) store_step(d);
        }
        if (iters - it == 2) {              // the last step of a task has nobody to publish to
            step_fwd<PR, PC, NW, 0, true, CHAIN>(xc, wy, ph0, w, d, e, d2, e2, xc.hin + it * (K::kHistRow * 4));
            ph0 ^= 1;
            if constexpr (MODE == kStoreSteps) store_step(d2);
            step_fwd<PR, PC, NW, 1, false, CHAIN>(xc, wy, ph1, w, d2, e2, d, e, xc.hin + (it + 1) * (K::kHistRow * 4));
            ph1 ^= 1;
        } else if (iters - it == 1) {
            step_fwd<PR, PC, NW, 0, false, CHAIN>(xc, wy, ph0, w, d, e, d2, e2, xc.hin + it * (K::kHistRow * 4));
            ph0 ^= 1;
        }
        CSPN_STAMP(xc, kTraceEvents - 2);
        cluster_arrive_relaxed();  // this CTA no longer reads its exchange buffers (paired with the wait above / after the loop)
        if (iters & 1) {
#pragma unroll
            for (int r = 0; r < PR; ++r)
#pragma unroll
                for (int j = 0; j < PC; ++j) d[r][j] = d2[r][j];
        }
        }   // MODE != kAdjoint

        // ---- epilogue: useful columns straight to global ------------------------------------------------
        float* out = prm.out + (size_t)bc * HW;
        const bool fan_out = MODE == kForward && (prm.n_peer != 0 || prm.out_mc != nullptr);   // fused gather (uniform)
        const int ux0 = prm.ux0[strip], ux1 = prm.ux1[strip];
        const int uy0 = GENERAL ? prm.uy0[band] : 0, uy1 = GENERAL ? prm.uy1[band] : H;   // uy1 <= H
        if (x_thr >= ux0 && x_thr < ux1) {
#pragma unroll
            for (int r = 0; r < PR; ++r) {
                const int y = y_thr + r;
                if (y >= uy0 && y < uy1) {
                    const float4 v = make_float4(d[r][0], d[r][1], d[r][2], d[r][3]);
                    if constexpr (MODE == kForward) {
                        __stcs(reinterpret_cast<float4*>(out + (size_t)y * W + x_thr), v);
                        if (fan_out) {
                            const size_t off = (size_t)bc * HW + (size_t)y * W + x_thr;
                            for (int e = 0; e < prm.n_peer; ++e)    // peer GPUs' gather buffers (NVLink stores)
                                __stcs(reinterpret_cast<float4*>(prm.out_peer[e] + off), v);
                            if (prm.out_mc)                         // NVLS: one store, replicated by the switch
                                asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(prm.out_mc + off),
                                             "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
                        }
                    } else {
                        *reinterpret_cast<float4*>(out + (size_t)y * W + x_thr) = v;   // read again by the next pass
                    }
                }
            }
        }
        if constexpr (CHAIN) {
            if (has_out) {      // uniform over the cluster: hand this CTA's rows of the recorded column to the next strip
                __syncthreads();                                  // every warp's history stores are in shared memory
                const size_t blk = ((size_t)strip * nq + qi) * csize + crank;
                float4* dst = reinterpret_cast<float4*>(prm.hist + blk * (size_t)(prm.iters * K::kHistRow));
                const float4* src = reinterpret_cast<const float4*>(hist_in + K::kHistBytes / sizeof(float));
                const int n16 = prm.iters * K::kHistRow / 4;
                for (int i = tid; i < n16; i += K::kThreads) __stcg(dst + i, src[i]);
                __syncthreads();
                // release is cumulative over what the barrier made visible to this thread: no separate fence
                if (tid == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(prm.flags + blk), "r"(1u) : "memory");
            }
        }
        CSPN_STAMP(xc, kTraceEvents - 1);
    }
    // No CTA may exit while a neighbour could still address its shared memory.
    if (!first) cluster_wait();
}

// ---- host side: configurations, planner, launch ---------------------------------------------------

struct KernelCfg {
    int PR, PC, NW;
    const void* fn[2][2];      // kForward: [general][norm_abs]
    const void* fn_steps[2];   // kStoreSteps [norm_abs]
    const void* fn_adj[2];     // kAdjoint    [norm_abs]
    const void* fn_chain[2][2];   // kForward with chained strips: [general][norm_abs]; null when the configuration has no such kernel
    size_t smem, smem_chain;
    int RB() const { return PR * NW; }
    int TW() const { return 32 * PC; }
};

template <int PR, int PC, int NW>
KernelCfg make_cfg() {
    return KernelCfg{PR, PC, NW,
                     {{(const void*)&cspn2d_cluster_kernel<PR, PC, NW, false, false>, (const void*)&cspn2d_cluster_kernel<PR, PC, NW, true, false>},
                      {(const void*)&cspn2d_cluster_kernel<PR, PC, NW, false, true>, (const void*)&cspn2d_cluster_kernel<PR, PC, NW, true, true>}},
                     {(const void*)&cspn2d_cluster_kernel<PR, PC, NW, false, true, kStoreSteps>,
                      (const void*)&cspn2d_cluster_kernel<PR, PC, NW, true, true, kStoreSteps>},
                     {(const void*)&cspn2d_cluster_kernel<PR, PC, NW, false, true, kAdjoint>,
                      (const void*)&cspn2d_cluster_kernel<PR, PC, NW, true, true, kAdjoint>},
                     {{nullptr, nullptr}, {nullptr, nullptr}},
                     Cfg<PR, PC, NW>::kSmemBytes, 0};
}
template <int PR, int PC, int NW>
KernelCfg make_cfg_chain() {
    KernelCfg k = make_cfg<PR, PC, NW>();
    k.fn_chain[0][0] = (const void*)&cspn2d_cluster_kernel<PR, PC, NW, false, false, kForward, true>;
    k.fn_chain[0][1] = (const void*)&cspn2d_cluster_kernel<PR, PC, NW, true, false, kForward, true>;
    k.fn_chain[1][0] = (const void*)&cspn2d_cluster_kernel<PR, PC, NW, false, true, kForward, true>;
    k.fn_chain[1][1] = (const void*)&cspn2d_cluster_kernel<PR, PC, NW, true, true, kForward, true>;
    k.smem_chain = Cfg<PR, PC, NW>::kSmemBytesChain;
    return k;
}

// The menu the planner picks from.  Register budget per pixel: 8 weights + value + second value set (c' is in shared
// memory); 8 warps (2 per SM sub-partition) may use 255 registers each -> up to 20 pixels per thread.
#ifdef CSPN_DEV_SINGLE
// developer build for offline SASS studies (tools/sass_loop.py on a 10-second compile): only the headline kernels
const std::vector<KernelCfg>& configs() {
    static const std::vector<KernelCfg> v = [] {
        KernelCfg k{5, 4, 8, {{nullptr, nullptr}, {nullptr, nullptr}}, {nullptr, nullptr}, {nullptr, nullptr}, {{nullptr, nullptr}, {nullptr, nullptr}},
                    Cfg<5, 4, 8>::kSmemBytes, Cfg<5, 4, 8>::kSmemBytesChain};
        k.fn[0][0] = (const void*)&cspn2d_cluster_kernel<5, 4, 8, false, false>;
        k.fn_chain[0][0] = (const void*)&cspn2d_cluster_kernel<5, 4, 8, false, false, kForward, true>;
        return std::vector<KernelCfg>{k};
    }();
    return v;
}
#else
const std::vector<KernelCfg>& configs() {
    static const std::vector<KernelCfg> v = {
        make_cfg_chain<5, 4, 8>(),   // 40 rows x 128 cols, 20 px/thread
        make_cfg_chain<4, 4, 8>(),   // 32 x 128
        make_cfg_chain<3, 4, 8>(),   // 24 x 128
        make_cfg<2, 4, 8>(),   // 16 x 128 (small images)
        make_cfg<5, 4, 4>(),   // 20 x 128 with 4 warps: two CTAs (of different tasks) fit one SM and de-phase each other
    };
    return v;
}
#endif

// One pass = one launch that advances every image by `iters` steps.
struct PassPlan {
    int cfg = -1, cs = 0, iters = 0, max_clusters = 0;
    bool chained = false;     // strips are processed left to right and hand their boundary column on (one-sided halos)
    int chain_lane = 0;
    int n_strips = 0, n_bands = 0;
    int tile_x0[kMaxStrips], ux0[kMaxStrips], ux1[kMaxStrips];
    int band_y0[kMaxBands], uy0[kMaxBands], uy1[kMaxBands];
    double cost = 0;
};
// The whole call: n_pass launches; the first n_long of them run `longp` (one step more), the rest `shortp`.
// Splitting N steps into passes trades one round trip of d through HBM (8 B/px, the kernel is nowhere near HBM-bound)
// for halos of N/n_pass instead of N columns: at N=48 a 128-column strip would keep only 32 useful columns.
struct Plan {
    int n_pass = 0, n_long = 0;
    PassPlan longp, shortp;
    double cost = 0;
    const PassPlan& pass(int i) const { return i < n_long ? longp : shortp; }
};

std::mutex g_mu;
unsigned long long* g_trace = nullptr;   // -DCSPN_TRACE builds: set through cspn_debug_set_trace
struct OccKey { int cfg, cs, dev, chained; };
std::vector<std::pair<OccKey, int>> g_occ_cache;
bool g_attr_set[16][16] = {};

int sm_count(int dev) {
    static int cached[16] = {};
    if (!cached[dev & 15]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { cudaGetLastError(); n = 132; }
        cached[dev & 15] = n;
    }
    return cached[dev & 15];
}

// how many clusters of `cs` CTAs of configuration `ci` can be co-resident on the device
int max_active_clusters(int ci, int cs, int dev, bool chained = false) {
    for (auto& e : g_occ_cache)
        if (e.first.cfg == ci && e.first.cs == cs && e.first.dev == dev && e.first.chained == (int)chained) return e.second;
    const KernelCfg& k = configs()[ci];
    if (chained && !k.fn_chain[0][0]) return 0;
    if (!g_attr_set[dev & 15][ci]) {
        const void* all[12] = {k.fn[0][0], k.fn[0][1], k.fn[1][0], k.fn[1][1], k.fn_steps[0], k.fn_steps[1], k.fn_adj[0], k.fn_adj[1],
                               k.fn_chain[0][0], k.fn_chain[0][1], k.fn_chain[1][0], k.fn_chain[1][1]};
        for (int i = 0; i < 12; ++i) {
            const void* f = all[i];
            if (!f) continue;
            if (cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(i >= 8 ? k.smem_chain : k.smem)) != cudaSuccess ||
                cudaFuncSetAttribute(f, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) {
                cudaGetLastError();
                return 0;
            }
        }
        g_attr_set[dev & 15][ci] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs * 64);
    cfg.blockDim = dim3(32 * k.NW);
    cfg.dynamicSmemBytes = chained ? k.smem_chain : k.smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cs;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, chained ? k.fn_chain[1][0] : k.fn[1][0], &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
    g_occ_cache.push_back({OccKey{ci, cs, dev, (int)chained}, n});
    return n;
}

// Chained cover of [0, L): tile i starts where tile i-1's useful range ends (its left neighbour column is handed over step
// by step), so only the RIGHT `halo` positions of a tile go stale; the last tile reaches the image border.
bool layout_1d_chained(int L, int T, int halo, int align, int min_useful, int max_n, int& n, int* t0, int* u0, int* u1) {
    n = 0;
    if (T >= L) return false;                                  // one tile: nothing to chain
    const int h = (halo + align - 1) / align * align;
    if (T - h < min_useful) return false;
    int u = 0;
    while (u < L) {
        if (n == max_n) return false;
        const int e = (u + T >= L) ? L : u + T - h;
        t0[n] = u; u0[n] = u; u1[n] = e;
        ++n;
        u = e;
    }
    return true;
}

// Cover [0, L) with tiles of T positions whose outer `halo` positions (rounded up to `align`) go stale during a pass:
// tile i starts at t0[i] (a multiple of `align`) and contributes the useful range [u0[i], u1[i]).  Tiles that touch the
// image border lose nothing on that side (zero padding is the reference's own boundary condition).
bool layout_1d(int L, int T, int halo, int align, int min_useful, int max_n, int& n, int* t0, int* u0, int* u1) {
    n = 0;
    if (T >= L) { t0[0] = 0; u0[0] = 0; u1[0] = L; n = 1; return true; }
    const int h = (halo + align - 1) / align * align;
    if (T - 2 * h < min_useful) return false;
    int u = 0;
    while (u < L) {
        if (n == max_n) return false;
        const int x0 = (u == 0) ? 0 : u - h;
        const int e = (x0 + T >= L) ? L : x0 + T - h;
        t0[n] = x0; u0[n] = u; u1[n] = e;
        ++n;
        u = e;
    }
    return true;
}

// Best (configuration, cluster size, strips, bands) for one pass of `iters` steps: minimises SM time per image.
// Deliberately independent of B and C, so the same image gets the same tiling (hence bit-identical results) whatever
// batch it is part of.  `dev` < 0: no device query (planning without a GPU): assume the H100 SXM occupancy table
// measured by tools/probe.cu.
bool plan_pass(int H, int W, int iters, int dev, int forced, bool chained, PassPlan& best) {
    static const int kProbe256[17] = {0, 132, 66, 39, 30, 22, 17, 15, 15, 9, 7, 7, 7, 7, 7, 7, 7};
    const char* fcs = getenv("CSPN_B200_FORCE_CS");   // developer hook for tuning runs (with CSPN_B200_FORCE_PASSES)
    const int forced_cs = fcs ? atoi(fcs) : 0;
    best.cfg = -1;
    const auto& cf = configs();
    const int n_sms = dev >= 0 ? sm_count(dev) : 132;
    for (int ci = 0; ci < (int)cf.size(); ++ci) {
        if (forced >= 0 && ci != forced) continue;
        const KernelCfg& k = cf[ci];
        PassPlan p;
        // columns: 4-aligned strip origins (TMA / float4), at least 16 useful columns per strip
        if (chained) {
            if (!k.fn_chain[0][0] || iters > kChainMaxIters) continue;
            if (!layout_1d_chained(W, k.TW(), iters, 4, 16, kMaxStrips, p.n_strips, p.tile_x0, p.ux0, p.ux1)) continue;
            p.chained = true;
            p.chain_lane = (k.TW() - (iters + 3) / 4 * 4) / 4 - 1;   // its 4th column is the one left of the next tile
        } else if (!layout_1d(W, k.TW(), iters, 4, 16, kMaxStrips, p.n_strips, p.tile_x0, p.ux0, p.ux1)) continue;
        const int cs_full = (H + k.RB() - 1) / k.RB();   // cluster height that needs no row halo
        for (int cs = 1; cs <= 16 && cs <= cs_full; ++cs) {
            if (forced_cs > 0 && cs != forced_cs) continue;
            // rows: one band when the cluster spans the image, else overlapping bands (images taller than 16 CTAs,
            // or a cluster size that fills the GPCs better)
            if (!layout_1d(H, cs * k.RB(), iters, 1, 8, kMaxBands, p.n_bands, p.band_y0, p.uy0, p.uy1)) continue;
            if (chained && p.n_bands > 1) continue;     // the recorded column is handed over per CTA row range: one band
            const int mac = dev >= 0 ? max_active_clusters(ci, cs, dev, chained) : kProbe256[cs];
            if (mac <= 0) continue;
            // tasks x per-task work / co-resident clusters.  Per-task work: 8 FMA per pixel and step plus a fixed part
            // (load, normalisation, store) worth ~15 steps (fit of the BASELINE configs[2] iteration sweep).
            // When a small configuration fits two CTAs per SM they share the SM's FMA pipe: count SMs, not CTAs.
            const int ctas_per_sm = (mac * cs + n_sms - 1) / n_sms;
            p.cost = (double)p.n_strips * p.n_bands * k.RB() * k.TW() * (8.0 * iters + 120.0) * ctas_per_sm / mac;
            // row bands re-load their halo rows and multiply the task count, which this model does not see, so a banded
            // plan has to win by a margin
            if (p.n_bands > 1) p.cost *= 1.15;
            // a chained task is longer (recorded column: loads, selects, predicated stores per step; hand-over)
            if (chained) p.cost *= 1.20;
            p.cfg = ci; p.cs = cs; p.max_clusters = mac; p.iters = iters;
            if (best.cfg < 0 || p.cost < best.cost) best = p;
        }
    }
    return best.cfg >= 0;
}

struct PlanKey { int H, W, iters, dev, forced, chained; };
std::vector<std::pair<PlanKey, Plan>> g_plan_cache;   // guarded by g_mu; a handful of shapes per process

// Picks the number of passes and each pass's tiling.  Caller holds g_mu.
bool make_plan(int H, int W, int iters, int dev, Plan& out, char* why, int why_len, bool chained = false) {
    if (W % 4 != 0) { snprintf(why, why_len, "W=%d is not a multiple of 4 (TMA row pitch / vector stores)", W); return false; }
    // developer hook for tuning runs: CSPN_B200_FORCE_CFG=<index into configs()>, CSPN_B200_FORCE_PASSES=<n>
    const char* force = getenv("CSPN_B200_FORCE_CFG");
    const int forced = force ? atoi(force) : -1;
    const char* fpass = getenv("CSPN_B200_FORCE_PASSES");
    const bool no_cache = (fpass && atoi(fpass) > 0) || getenv("CSPN_B200_FORCE_CS") != nullptr;
    const int forced_passes = fpass ? atoi(fpass) : 0;
    for (auto& e : g_plan_cache)
        if (e.first.H == H && e.first.W == W && e.first.iters == iters && e.first.dev == dev && e.first.forced == forced &&
            e.first.chained == (int)chained && !no_cache) { out = e.second; return true; }
    Plan best;
    best.n_pass = 0;
    const int max_pass = iters < kMaxPasses ? iters : kMaxPasses;
    for (int P = 1; P <= max_pass; ++P) {
        if (forced_passes > 0 && P != forced_passes) continue;
        Plan c;
        c.n_pass = P;
        c.n_long = iters % P;
        const int a = iters / P;
        if (!plan_pass(H, W, a, dev, forced, chained, c.shortp)) continue;
        if (c.n_long > 0 && !plan_pass(H, W, a + 1, dev, forced, chained, c.longp)) continue;
        c.cost = (P - c.n_long) * c.shortp.cost + (c.n_long > 0 ? c.n_long * c.longp.cost : 0.0);
        if (best.n_pass == 0 || c.cost < best.cost) best = c;
        // more passes only pay while the halo shrinks faster than the fixed per-task part grows
        if (best.n_pass > 0 && P >= 2 * best.n_pass + 2) break;
    }
    if (best.n_pass == 0) {
        snprintf(why, why_len, "no cluster configuration covers H=%d W=%d iters=%d", H, W, iters);
        return false;
    }
    if (!no_cache) {
        if (g_plan_cache.size() >= 64) g_plan_cache.erase(g_plan_cache.begin());
        g_plan_cache.push_back({PlanKey{H, W, iters, dev, forced, (int)chained}, best});
    }
    out = best;
    return true;
}

int current_device_or_none() {
    int ndev = 0, dev = -1;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { cudaGetLastError(); return -1; }
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return -1; }
    return dev;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int get_encode() {
    if (g_encode) return CSPN_OK;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CSPN_CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !fn) {
        set_error("cuTensorMapEncodeTiled not available from the driver");
        return CSPN_ERR_CUDA;
    }
    g_encode = (EncodeTiledFn)fn;
    return CSPN_OK;
}

}  // namespace

#ifdef CSPN_TRACE
// developer hook of the tracing build only (not declared in include/cspn_b200.h): device buffer of
// kTraceTasks*16*8*kTraceEvents 64-bit stamps, or null to stop tracing
extern "C" __attribute__((visibility("default"))) void cspn_debug_set_trace(void* buf) { g_trace = static_cast<unsigned long long*>(buf); }
extern "C" __attribute__((visibility("default"))) int cspn_debug_trace_events() { return kTraceEvents; }
#endif

bool cluster2d_supported(const Problem2D& p, char* why, int why_len) {
    if (p.iters <= 0) { snprintf(why, why_len, "iters == 0"); return false; }
    if ((reinterpret_cast<uintptr_t>(p.guidance) | reinterpret_cast<uintptr_t>(p.blur) | reinterpret_cast<uintptr_t>(p.sparse) |
         reinterpret_cast<uintptr_t>(p.out)) & 15) {
        snprintf(why, why_len, "tensor base pointers must be 16-byte aligned");
        return false;
    }
    if ((long)p.B * p.gch > 2147483647L) { snprintf(why, why_len, "B*gch too large"); return false; }
    const int dev = current_device_or_none();
    std::lock_guard<std::mutex> lock(g_mu);
    Plan plan;
    if (!make_plan(p.H, p.W, p.iters, dev, plan, why, why_len)) return false;
    for (int i = 0; i < 2; ++i) {
        const PassPlan& pp = i ? plan.shortp : plan.longp;
        if (pp.cfg >= 0 && (long)p.B * p.C * pp.n_strips * pp.n_bands > 2147483647L) {
            snprintf(why, why_len, "too many tasks");
            return false;
        }
    }
    return true;
}

namespace {
// Chained strips need, per pass, one history block per (strip boundary, image-channel, CTA of the cluster) and a flag each.
struct ChainWs { size_t hist_bytes = 0, flag_bytes = 0; size_t total() const { return hist_bytes + flag_bytes; } };
ChainWs chain_ws(const Plan& plan, long BC) {
    ChainWs w;
    for (int i = 0; i < 2; ++i) {
        const PassPlan& pp = i ? plan.shortp : plan.longp;
        if (pp.cfg < 0 || !pp.chained || (i == 0 && plan.n_long == 0)) continue;
        const size_t blocks = (size_t)(pp.n_strips - 1) * BC * pp.cs;
        const size_t hb = (blocks * pp.iters * configs()[pp.cfg].NW * 8 * sizeof(float) + 255) / 256 * 256;
        const size_t fb = (blocks * sizeof(unsigned) + 255) / 256 * 256;
        if (hb > w.hist_bytes) w.hist_bytes = hb;
        if (fb > w.flag_bytes) w.flag_bytes = fb;
    }
    return w;
}
// The plan a call with B*C image-channels uses when it is given enough workspace: chained strips pay when every cluster
// has at least two rounds of tasks (a task's left neighbour strip is then long finished) and the planner's model says so.
// CSPN_B200_CHAIN=0 never chains, =1 chains whenever a chained plan exists (tests, tuning).  Caller holds g_mu.
bool choose_plan(int H, int W, int iters, int dev, long BC, Plan& plan, bool& chained, char* why, int why_len) {
    chained = false;
    if (!make_plan(H, W, iters, dev, plan, why, why_len)) return false;
    const char* ce = getenv("CSPN_B200_CHAIN");
    if (ce && ce[0] == '0') return true;
    Plan cp;
    char why2[200] = "";
    if (!make_plan(H, W, iters, dev, cp, why2, sizeof(why2), true)) return true;
    const bool forced = ce && ce[0] == '1';
    if (forced || (BC >= 2L * cp.shortp.max_clusters && cp.cost < plan.cost)) { plan = cp; chained = true; }
    return true;
}
}  // namespace

// Passes after the first read the previous pass's result: one extra d-sized buffer (passes alternate between it and
// `out`, ending in `out`).  Chained strips add their history blocks and flags; a call that gets less workspace than that
// (but enough for the passes) runs the unchained plan.
size_t cluster2d_workspace_bytes(int B, int C, int H, int W, int iters) {
    if (iters <= 0) return 0;
    const int dev = current_device_or_none();
    std::lock_guard<std::mutex> lock(g_mu);
    Plan plan;
    char why[200] = "";
    if (!make_plan(H, W, iters, dev, plan, why, sizeof(why))) return 0;
    const size_t d_bytes = (size_t)B * C * H * W * sizeof(float);
    size_t need = plan.n_pass > 1 ? d_bytes : 0;
    Plan cp;
    bool chained = false;
    if (choose_plan(H, W, iters, dev, (long)B * C, cp, chained, why, sizeof(why)) && chained) {
        const size_t c = (cp.n_pass > 1 ? d_bytes : 0) + chain_ws(cp, (long)B * C).total();
        if (c > need) need = c;
    }
    return need;
}

int cluster2d_describe(int B, int C, int H, int W, int iters, char* buf, int len) {
    const int dev = current_device_or_none();
    std::lock_guard<std::mutex> lock(g_mu);
    Plan plan;
    char why[200] = "";
    bool chained = false;
    if (!choose_plan(H, W, iters, dev, (long)B * C, plan, chained, why, sizeof(why))) return snprintf(buf, len, "cluster: unsupported (%s)", why);
    const PassPlan& pp = plan.shortp;
    const KernelCfg& k = configs()[pp.cfg];
    long useful_x = 0, useful_y = 0;
    for (int i = 0; i < pp.n_strips; ++i) useful_x += pp.ux1[i] - pp.ux0[i];
    for (int i = 0; i < pp.n_bands; ++i) useful_y += pp.uy1[i] - pp.uy0[i];
    char passes[96] = "";
    if (plan.n_pass > 1)
        snprintf(passes, sizeof(passes), "%d passes (%d x %d + %d x %d steps), ", plan.n_pass, plan.n_long, pp.iters + 1,
                 plan.n_pass - plan.n_long, pp.iters);
    return snprintf(buf, len,
                    "cluster: %spatch %dx%d px/thread, %d warps -> CTA tile %d rows x %d cols, cluster of %d CTAs (%d rows), "
                    "%d %sstrip(s) x %d band(s)/image, %ld tasks, %d co-resident clusters, lane efficiency %.2f, smem %zu B",
                    passes, k.PR, k.PC, k.NW, k.RB(), k.TW(), pp.cs, pp.cs * k.RB(), pp.n_strips, chained ? "chained " : "", pp.n_bands,
                    (long)B * C * pp.n_strips * pp.n_bands, pp.max_clusters,
                    (double)useful_x * useful_y / ((double)pp.n_strips * k.TW() * pp.n_bands * pp.cs * k.RB()),
                    chained ? k.smem_chain : k.smem);
}

// Machine-readable plan (tests/test_plan_cpu.py replays it on the CPU oracle): every pass with its tile geometry.
int cluster2d_plan_json(int H, int W, int iters, int chained, char* buf, int len) {
    const int dev = current_device_or_none();
    std::lock_guard<std::mutex> lock(g_mu);
    Plan plan;
    char why[200] = "";
    if (!make_plan(H, W, iters, dev, plan, why, sizeof(why), chained != 0)) return snprintf(buf, len, "{\"supported\": false, \"why\": \"%s\"}", why);
    int n = snprintf(buf, len, "{\"supported\": true, \"chained\": %s, \"passes\": [", chained ? "true" : "false");
    for (int part = 0; part < 2; ++part) {
        const int count = part == 0 ? plan.n_long : plan.n_pass - plan.n_long;
        if (count == 0) continue;
        const PassPlan& pp = part == 0 ? plan.longp : plan.shortp;
        const KernelCfg& k = configs()[pp.cfg];
        auto put = [&](const char* fmt, auto... a) { if (n < len) n += snprintf(buf + n, len - n, fmt, a...); };
        put("%s{\"count\": %d, \"iters\": %d, \"PR\": %d, \"NW\": %d, \"RB\": %d, \"TW\": %d, \"cs\": %d, \"max_clusters\": %d, \"strips\": [",
            (part == 1 && plan.n_long > 0) ? ", " : "", count, pp.iters, k.PR, k.NW, k.RB(), k.TW(), pp.cs, pp.max_clusters);
        for (int i = 0; i < pp.n_strips; ++i) put("%s[%d, %d, %d]", i ? ", " : "", pp.tile_x0[i], pp.ux0[i], pp.ux1[i]);
        put("%s", "], \"bands\": [");
        for (int i = 0; i < pp.n_bands; ++i) put("%s[%d, %d, %d]", i ? ", " : "", pp.band_y0[i], pp.uy0[i], pp.uy1[i]);
        put("%s", "]}");
    }
    if (n < len) n += snprintf(buf + n, len - n, "]}");
    return n;
}

namespace {

int plan_for_launch(const Problem2D& p, Plan& plan) {
    int dev = 0;
    CSPN_CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_mu);
    char why[200] = "";
    if (!make_plan(p.H, p.W, p.iters, dev, plan, why, sizeof(why))) {
        set_error("cluster kernel unsupported: %s", why);
        return CSPN_ERR_UNSUPPORTED;
    }
    return get_encode();
}

// One pass = one launch of `fn` with plan `pp`.  `start` plays the role of blur_depth (kAdjoint: lambda's start value),
// `init` continues from an earlier pass (kForward / kStoreSteps), `iter_out` / `iter_stride` say where every step but
// the last is written (kStoreSteps / kAdjoint), the last step goes to `out`.
// Tiled 3D tensor map over `planes` row-major (H, W) fp32 planes, box (bx, by, 1).  The descriptor is a pure function of
// (base pointer, shape, box): serving loops call with the same buffers again and again, so the last few encodings are
// kept (the driver call costs microseconds, which is what a 1-image problem lasts).
int tensor_map_3d(const float* base, int W, int H, int planes, int bx, int by, CUtensorMap& tm) {
    struct MapKey { const void* base; int W, H, planes, bx, by; };
    struct MapEntry { MapKey key; CUtensorMap tm; };
    constexpr int kCached = 16;
    static MapEntry cache[kCached];
    static int n_cached = 0, next_slot = 0;
    const MapKey key{base, W, H, planes, bx, by};
    {
        std::lock_guard<std::mutex> lock(g_mu);
        for (int i = 0; i < n_cached; ++i) {
            const MapKey& c = cache[i].key;
            if (c.base == key.base && c.W == key.W && c.H == key.H && c.planes == key.planes && c.bx == key.bx && c.by == key.by) {
                tm = cache[i].tm;
                return CSPN_OK;
            }
        }
    }
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)planes};
    const cuuint64_t strides[2] = {(cuuint64_t)W * sizeof(float), (cuuint64_t)W * H * sizeof(float)};
    const cuuint32_t estr[3] = {1, 1, 1};
    const cuuint32_t box[3] = {(cuuint32_t)bx, (cuuint32_t)by, 1};
    CUresult cr = g_encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (W=%d H=%d planes=%d box=%dx%d)", (int)cr, W, H, planes, bx, by);
        return CSPN_ERR_CUDA;
    }
    std::lock_guard<std::mutex> lock(g_mu);
    cache[next_slot] = MapEntry{key, tm};
    next_slot = (next_slot + 1) % kCached;
    if (n_cached < kCached) ++n_cached;
    return CSPN_OK;
}

struct Scatter { float* const* peer = nullptr; int n_peer = 0; float* mc = nullptr; };
struct ChainBuf { float* hist = nullptr; unsigned* flags = nullptr; size_t flag_bytes = 0; };   // chained passes only

int launch_pass(const Problem2D& p, const PassPlan& pp, const void* fn, const float* start, const float* init, float* out,
                float* iter_out, long long iter_stride, cudaStream_t stream, const Scatter& sc = Scatter(),
                const ChainBuf& cb = ChainBuf()) {
    const KernelCfg& k = configs()[pp.cfg];
    const bool chained = cb.hist != nullptr;
    // guidance as a 3D tensor (W, H, B*gch); one box = (TW + 8, RB, 1) floats of one channel plane (4 apron columns per
    // side).  blur / sparse as (W, H, planes) with (TW, RB, 1) boxes: only ever PREFETCHED into L2 through their maps.
    CUtensorMap tm, tm_blur, tm_sparse;
    int rc = tensor_map_3d(p.guidance, p.W, p.H, p.B * p.gch, k.TW() + 8, k.RB(), tm);
    if (rc != CSPN_OK) return rc;
    rc = tensor_map_3d(start, p.W, p.H, p.B * p.C, k.TW(), k.RB(), tm_blur);
    if (rc != CSPN_OK) return rc;
    if (p.sparse) {
        rc = tensor_map_3d(p.sparse, p.W, p.H, p.B, k.TW(), k.RB(), tm_sparse);
        if (rc != CSPN_OK) return rc;
    } else {
        tm_sparse = tm_blur;      // never dereferenced (prm.sparse == nullptr)
    }
    ClusterParams prm;
    prm.blur = start; prm.init = init; prm.sparse = p.sparse; prm.out = out;
    prm.iter_out = iter_out; prm.iter_stride = iter_stride;
    prm.C = p.C; prm.H = p.H; prm.W = p.W; prm.gch = p.gch; prm.iters = pp.iters; prm.norm_abs = p.norm_abs;
    prm.n_strips = pp.n_strips;
    prm.n_bands = pp.n_bands;
    prm.trace = g_trace;
    prm.hist = cb.hist; prm.flags = cb.flags; prm.chain_lane = pp.chain_lane;
    {
        // group size: at least 1.5 x the co-resident clusters, the groups as equal as possible.  A strip's left neighbour then
        // runs at least one full round of clusters earlier, so its flag is normally set when it is first looked at, yet recently
        // enough that the guidance columns the two tiles share still come from L2 instead of DRAM.  CSPN_B200_CHAIN_GROUP
        // overrides (0 = one group).
        const long nq_all = (long)p.B * p.C * pp.n_bands;
        long min_g = pp.max_clusters + (pp.max_clusters + 1) / 2;
        if (const char* e = getenv("CSPN_B200_CHAIN_GROUP")) min_g = atol(e) > 0 ? atol(e) : nq_all;
        long n_groups = min_g > 0 ? nq_all / min_g : 1;
        if (n_groups < 1) n_groups = 1;
        prm.chain_group = (int)(nq_all / n_groups);
    }
    prm.n_peer = sc.n_peer;
    for (int i = 0; i < 7; ++i) prm.out_peer[i] = i < sc.n_peer ? sc.peer[i] : nullptr;
    prm.out_mc = sc.mc;
    const long tasks = (long)p.B * p.C * pp.n_strips * pp.n_bands;
    if (tasks > 2147483647L) { set_error("too many tasks"); return CSPN_ERR_UNSUPPORTED; }
    prm.n_tasks = (int)tasks;
    for (int i = 0; i < kMaxStrips; ++i) {
        const bool in = i < pp.n_strips;
        prm.tile_x0[i] = in ? pp.tile_x0[i] : 0; prm.ux0[i] = in ? pp.ux0[i] : 0; prm.ux1[i] = in ? pp.ux1[i] : 0;
    }
    for (int i = 0; i < kMaxBands; ++i) {
        const bool in = i < pp.n_bands;
        prm.band_y0[i] = in ? pp.band_y0[i] : 0; prm.uy0[i] = in ? pp.uy0[i] : 0; prm.uy1[i] = in ? pp.uy1[i] : 0;
    }
    // persistent clusters: as many as fit on the device at once, each looping over tasks
    const long n_clusters = tasks < pp.max_clusters ? tasks : pp.max_clusters;

    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(n_clusters * pp.cs));
    cfg.blockDim = dim3(32 * k.NW);
    cfg.dynamicSmemBytes = chained ? k.smem_chain : k.smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = pp.cs;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    if (chained) {
        // a task spins on the flag of its left neighbour strip, which another cluster sets: every cluster of the grid must be
        // resident (the grid is sized by the occupancy query; a cooperative launch makes that a guarantee, not a hope)
        // (developer hook CSPN_B200_COOP=0: plain launch, for Nsight Compute -- its replay of a cooperative launch drops
        // the cluster dimension; under the profiler kernels run alone, so residency holds anyway)
        const char* coop = getenv("CSPN_B200_COOP");
        if (!(coop && coop[0] == '0')) {
            at[1].id = cudaLaunchAttributeCooperative;
            at[1].val.cooperative = 1;
            cfg.numAttrs = 2;
        }
        CSPN_CUDA_TRY(cudaMemsetAsync(cb.flags, 0, cb.flag_bytes, stream));
    }
    void* args[4] = {(void*)&tm, (void*)&tm_blur, (void*)&tm_sparse, (void*)&prm};
    CSPN_CUDA_TRY(cudaLaunchKernelExC(&cfg, fn, args));
    return CSPN_OK;
}

}  // namespace

int cluster2d_forward(const Problem2D& p, void* ws, size_t ws_bytes, cudaStream_t stream, int* launches, float* const* peer_out,
                      int n_peer, float* mc_out) {
    Plan plan;
    int rc = plan_for_launch(p, plan);
    if (rc != CSPN_OK) return rc;
    const size_t d_bytes = (size_t)p.B * p.C * p.H * p.W * sizeof(float);
    // chained strips when the planner wants them and the caller's workspace holds their history blocks
    ChainBuf cb;
    {
        int dev = 0;
        CSPN_CUDA_TRY(cudaGetDevice(&dev));
        std::lock_guard<std::mutex> lock(g_mu);
        Plan cp;
        bool chained = false;
        char why[200] = "";
        if (choose_plan(p.H, p.W, p.iters, dev, (long)p.B * p.C, cp, chained, why, sizeof(why)) && chained) {
            const ChainWs cw = chain_ws(cp, (long)p.B * p.C);
            const size_t base = cp.n_pass > 1 ? d_bytes : 0;
            if (ws && ws_bytes >= base + cw.total() && (reinterpret_cast<uintptr_t>(ws) & 15) == 0 && d_bytes % 16 == 0) {
                plan = cp;
                cb.hist = reinterpret_cast<float*>(static_cast<char*>(ws) + base);
                cb.flags = reinterpret_cast<unsigned*>(static_cast<char*>(ws) + base + cw.hist_bytes);
                cb.flag_bytes = cw.flag_bytes;
            }
        }
    }
    if (plan.n_pass > 1 && (!ws || ws_bytes < d_bytes)) {
        set_error("cluster path splits %d steps into %d passes and needs %zu workspace bytes, got %zu", p.iters, plan.n_pass,
                  d_bytes, ws ? ws_bytes : (size_t)0);
        return CSPN_ERR_WORKSPACE;
    }
    const float* prev = nullptr;   // result of the previous pass
    for (int ip = 0; ip < plan.n_pass; ++ip) {
        const PassPlan& pp = plan.pass(ip);
        // passes alternate between the workspace and `out` such that the last one lands in `out`
        float* dst = ((plan.n_pass - 1 - ip) & 1) ? static_cast<float*>(ws) : p.out;
        const bool general = pp.n_bands > 1 || prev != nullptr;
        Scatter sc;
        if (ip == plan.n_pass - 1) { sc.peer = peer_out; sc.n_peer = n_peer; sc.mc = mc_out; }   // only the final result travels
        const KernelCfg& kc = configs()[pp.cfg];
        rc = launch_pass(p, pp, (pp.chained ? kc.fn_chain : kc.fn)[general ? 1 : 0][p.norm_abs ? 1 : 0], p.blur, prev, dst, nullptr, 0, stream, sc,
                         pp.chained ? cb : ChainBuf());
        if (rc != CSPN_OK && pp.chained && ip == 0) {
            // the cooperative launch was refused (the grid cannot be made resident as a whole: SM partitioning, MPS limits, ...):
            // nothing has run yet, so take the unchained plan, which needs no residency guarantee
            cudaGetLastError();
            clear_error();
            rc = plan_for_launch(p, plan);
            if (rc != CSPN_OK) return rc;
            if (plan.n_pass > 1 && (!ws || ws_bytes < d_bytes)) { set_error("workspace too small for the unchained plan"); return CSPN_ERR_WORKSPACE; }
            cb = ChainBuf();
            ip = -1;
            prev = nullptr;
            continue;
        }
        if (rc != CSPN_OK) return rc;
        ++*launches;
        prev = dst;
    }
    return CSPN_OK;
}

// The forward again, keeping every iterate: steps[t] = d_{t+1} for t = 0..N-1 (planes of B*C*H*W floats).
int cluster2d_forward_steps(const Problem2D& p, float* steps, cudaStream_t stream, int* launches) {
    Plan plan;
    int rc = plan_for_launch(p, plan);
    if (rc != CSPN_OK) return rc;
    const long long n = (long long)p.B * p.C * p.H * p.W;
    int done = 0;
    for (int ip = 0; ip < plan.n_pass; ++ip) {
        const PassPlan& pp = plan.pass(ip);
        rc = launch_pass(p, pp, configs()[pp.cfg].fn_steps[p.norm_abs ? 1 : 0], p.blur, done ? steps + (done - 1) * n : nullptr,
                         steps + (done + pp.iters - 1) * n, steps + done * n, n, stream);
        if (rc != CSPN_OK) return rc;
        ++*launches;
        done += pp.iters;
    }
    return CSPN_OK;
}

// The adjoint sweep: lam[t] = lambda_t for t = N-1 .. 0, starting from lambda_N = grad_out.
int cluster2d_adjoint_steps(const Problem2D& p, const float* grad_out, float* lam, cudaStream_t stream, int* launches) {
    Plan plan;
    int rc = plan_for_launch(p, plan);
    if (rc != CSPN_OK) return rc;
    const long long n = (long long)p.B * p.C * p.H * p.W;
    const int N = p.iters;
    int done = 0;   // adjoint steps taken so far: lambda_{N-done} is the current state
    for (int ip = 0; ip < plan.n_pass; ++ip) {
        const PassPlan& pp = plan.pass(ip);
        rc = launch_pass(p, pp, configs()[pp.cfg].fn_adj[p.norm_abs ? 1 : 0], done ? lam + (long long)(N - done) * n : grad_out, nullptr,
                         lam + (long long)(N - done - pp.iters) * n, lam + (long long)(N - done - 1) * n, -n, stream);
        if (rc != CSPN_OK) return rc;
        ++*launches;
        done += pp.iters;
    }
    return CSPN_OK;
}

}  // namespace cspn
