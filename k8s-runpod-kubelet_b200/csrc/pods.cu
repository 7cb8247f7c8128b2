// pods.cu -- the pod-requirement table: the five pod columns of every tracked pod, kept on each GPU and indexed by
// the slot ids the Provider already gives the status table, so that a pending-pod tick (processPendingPods,
// kubelet.go:747-814) uploads 4 bytes of slot id per pod instead of the 21 bytes of its columns.
//
// Kernels:
//   k_pod_fill      every row := the columns of a pod with no annotations (rpk_pods_reset)
//   k_pod_seed      row slots[i] := element i of each staged column; a NULL column writes its default (rpk_pods_seed_slots)
//   k_pod_gather    compact columns of one rpk_select_slots sub-batch, or of one rpk_select_slots_device* call: element
//                   i := row slots[i] of the table, written into the lane's pod-column buffers, which the select kernels
//                   then read as rpk_select's uploaded ones
// The host entry points check every slot against the table's N before its upload.  The device entry points cannot, so
// an entry outside [0, N) is defined here: the seed skips it, and the gather writes a row with cloud byte kCloudNone,
// which every select path finishes as "neither cloud" (runpod_client.go:469-475): -1 and five -1.  No caller input
// can make these kernels touch memory outside the table.
#include <algorithm>

#include "rpk_internal.cuh"

namespace rpk {

constexpr int kPodThreads = 256;
constexpr int32_t kDefaultMemGb = 16;  // extractGPUMemory("") (runpod_client.go:1182)
constexpr uint8_t kCloudNone = 2;      // neither RPK_CLOUD_SECURE nor RPK_CLOUD_COMMUNITY: no offer is feasible

__global__ void k_pod_fill(PodRows t, uint32_t N) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
        t.mem[i] = kDefaultMemGb; t.vcpu[i] = 0; t.ram[i] = 0; t.max_price[i] = RPK_DEFAULT_MAX_PRICE; t.cloud[i] = RPK_CLOUD_SECURE;
    }
}

__global__ void k_pod_seed(PodRows t, uint32_t N, uint32_t n, const uint32_t* __restrict__ slots, PodCols in) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s >= N) return;
    t.mem[s] = in.req_mem[i];
    t.vcpu[s] = in.req_vcpu ? in.req_vcpu[i] : 0;
    t.ram[s] = in.req_ram ? in.req_ram[i] : 0;
    t.max_price[s] = in.max_price ? in.max_price[i] : RPK_DEFAULT_MAX_PRICE;
    t.cloud[s] = in.cloud ? in.cloud[i] : (uint8_t)RPK_CLOUD_SECURE;
}

__global__ void k_pod_gather(PodRows t, uint32_t N, uint32_t n, const uint32_t* __restrict__ slots, PodRows out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s >= N) {  // a row nothing matches; the other columns hold a pod with no annotations
        out.mem[i] = kDefaultMemGb; out.vcpu[i] = 0; out.ram[i] = 0; out.max_price[i] = RPK_DEFAULT_MAX_PRICE; out.cloud[i] = kCloudNone;
        return;
    }
    out.mem[i] = __ldg(t.mem + s); out.vcpu[i] = __ldg(t.vcpu + s); out.ram[i] = __ldg(t.ram + s);
    out.max_price[i] = __ldg(t.max_price + s); out.cloud[i] = __ldg(t.cloud + s);
}

int launch_pod_fill(const PodRows& t, uint32_t N, int sm_count, cudaStream_t st) {
    if (N == 0) return 0;
    const uint32_t blocks = std::min<uint32_t>((N + kPodThreads - 1) / kPodThreads, (uint32_t)sm_count * 8);
    k_pod_fill<<<blocks, kPodThreads, 0, st>>>(t, N);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_seed(const PodRows& t, uint32_t N, uint32_t n, const uint32_t* d_slots, const PodCols& in, cudaStream_t st) {
    if (n == 0) return 0;
    k_pod_seed<<<(n + kPodThreads - 1) / kPodThreads, kPodThreads, 0, st>>>(t, N, n, d_slots, in);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

int launch_pod_gather(const PodRows& t, uint32_t N, uint32_t n, const uint32_t* d_slots, const PodRows& out, cudaStream_t st) {
    if (n == 0) return 0;
    k_pod_gather<<<(n + kPodThreads - 1) / kPodThreads, kPodThreads, 0, st>>>(t, N, n, d_slots, out);
    RPK_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace rpk
