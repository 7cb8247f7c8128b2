// explain.cu -- rpk_explain / rpk_explain_slots: for every pod row, what rules out each offer of the resident table
// (include/rpk.h, rpk_explanation).  The select keeps at most five feasible offers and says nothing about the others,
// so this is a P x G grid of its own.
//
// Kernel:
//   k_explain   one row per thread, 256 rows per CTA.  For each cloud view c that some row of the tile selects from, the
//               CTA walks the offered prefix of v_wide[c] (price order, ties by offer index) in chunks of kExplainChunk
//               offers staged in shared memory: each offer is loaded from global memory once per CTA and read by every
//               row of the tile as a shared-memory broadcast.  The counters live in registers.  The price test is a
//               prefix of the view: one binary search of v_price per row gives the first position whose price is not
//               below the row's bound (IEEE; a NaN bound gives 0), so the walk compares positions, not doubles.  Because
//               the walk is in price order, nearest[r] is the first offer failing r alone.  A CTA that has no row of
//               cloud c does not walk view c, and rows of neither cloud are finished without a walk.  The rows' results
//               are staged in shared memory and written out as one coalesced copy.
#include "rpk_internal.cuh"

namespace rpk {

constexpr int kExplainThreads = 256;
constexpr uint32_t kExplainChunk = 1024;  // offers staged per pass: 16 KB of int4
constexpr uint32_t kExplainWords = sizeof(rpk_explanation) / 4;
static_assert(sizeof(rpk_explanation) == 56, "rpk_explanation is 14 words");
static_assert(kExplainChunk * sizeof(int4) >= kExplainThreads * sizeof(rpk_explanation), "the output stage reuses the offer stage");

// length of the offered prefix of a view: the unoffered offers and the padding sit at its tail with offer index -1
__device__ uint32_t offered_len(const int4* __restrict__ wide, uint32_t G) {
    uint32_t lo = 0, hi = G;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(&wide[mid].w) >= 0) lo = mid + 1; else hi = mid; }
    return lo;
}

// first position of the offered prefix [0, n) whose price is not below mx (the prices there are ascending and > 0)
__device__ uint32_t price_cut(const double* __restrict__ price, uint32_t n, double mx) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(price + mid) < mx) lo = mid + 1; else hi = mid; }
    return lo;
}

__global__ void __launch_bounds__(kExplainThreads) k_explain(ExplainArgs a) {
    __shared__ int4 stage[kExplainChunk];
    __shared__ uint32_t n_off[2];
    const uint32_t row0 = blockIdx.x * kExplainThreads, row = row0 + threadIdx.x;
    int c = -1;
    int32_t rm = 0, rv = 0, rr = 0;
    double mx = RPK_DEFAULT_MAX_PRICE;
    if (row < a.P) {
        const uint8_t cb = a.rows.cloud ? a.rows.cloud[row] : (uint8_t)RPK_CLOUD_SECURE;
        c = cb == RPK_CLOUD_SECURE ? 0 : cb == RPK_CLOUD_COMMUNITY ? 1 : -1;
        rm = a.rows.req_mem[row];
        rv = a.rows.req_vcpu ? a.rows.req_vcpu[row] : 0;
        rr = a.rows.req_ram ? a.rows.req_ram[row] : 0;
        mx = a.rows.max_price ? a.rows.max_price[row] : RPK_DEFAULT_MAX_PRICE;
    }
    const bool any0 = __syncthreads_or(c == 0) != 0, any1 = __syncthreads_or(c == 1) != 0;
    if (threadIdx.x < 2 && (threadIdx.x == 0 ? any0 : any1)) n_off[threadIdx.x] = offered_len(threadIdx.x == 0 ? a.wide[0] : a.wide[1], a.G);
    __syncthreads();

    uint32_t n = 0, cut = 0, feas = 0, fail_mem = 0, fail_vcpu = 0, fail_ram = 0;
    uint32_t only_price = 0, only_mem = 0, only_vcpu = 0, only_ram = 0;
    int32_t near_price = -1, near_mem = -1, near_vcpu = -1, near_ram = -1;
#pragma unroll 1
    for (int v = 0; v < 2; ++v) {
        if (!(v == 0 ? any0 : any1)) continue;
        const int4* wide = v == 0 ? a.wide[0] : a.wide[1];  // (a constant index keeps the arguments out of local memory)
        const uint32_t nv = n_off[v];
        const bool mine = c == v;
        if (mine) { n = nv; cut = price_cut(v == 0 ? a.price[0] : a.price[1], nv, mx); }
        for (uint32_t base = 0; base < nv; base += kExplainChunk) {
            const uint32_t m = min(kExplainChunk, nv - base);
            for (uint32_t i = threadIdx.x; i < m; i += kExplainThreads) stage[i] = __ldg(wide + base + i);
            __syncthreads();
            if (mine) {
#pragma unroll 4
                for (uint32_t j = 0; j < m; ++j) {
                    const int4 o = stage[j];
                    const bool fp = base + j >= cut, fm = o.x < rm, fv = o.y < rv, fr = o.z < rr;
                    const uint32_t nf = (uint32_t)fp + (uint32_t)fm + (uint32_t)fv + (uint32_t)fr;
                    feas += nf == 0;
                    fail_mem += fm; fail_vcpu += fv; fail_ram += fr;
                    if (nf == 1) {
                        only_price += fp; only_mem += fm; only_vcpu += fv; only_ram += fr;
                        if (fp && near_price < 0) near_price = o.w;
                        if (fm && near_mem < 0) near_mem = o.w;
                        if (fv && near_vcpu < 0) near_vcpu = o.w;
                        if (fr && near_ram < 0) near_ram = o.w;
                    }
                }
            }
            __syncthreads();
        }
    }

    // the tile's results through the (free) stage, then one coalesced copy
    uint32_t* sw = reinterpret_cast<uint32_t*>(stage) + threadIdx.x * kExplainWords;
    sw[0] = feas; sw[1] = a.G - n; sw[2] = n - cut; sw[3] = fail_mem; sw[4] = fail_vcpu; sw[5] = fail_ram;
    sw[6] = only_price; sw[7] = only_mem; sw[8] = only_vcpu; sw[9] = only_ram;
    sw[10] = (uint32_t)near_price; sw[11] = (uint32_t)near_mem; sw[12] = (uint32_t)near_vcpu; sw[13] = (uint32_t)near_ram;
    __syncthreads();
    const uint32_t rows = min((uint32_t)kExplainThreads, a.P - row0);
    uint32_t* out = reinterpret_cast<uint32_t*>(a.out + row0);
    for (uint32_t i = threadIdx.x; i < rows * kExplainWords; i += kExplainThreads) out[i] = reinterpret_cast<const uint32_t*>(stage)[i];
}

int launch_explain(const ExplainArgs& a, cudaStream_t st) {
    if (a.P == 0) return 0;
    k_explain<<<(a.P + kExplainThreads - 1) / kExplainThreads, kExplainThreads, 0, st>>>(a);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace rpk
