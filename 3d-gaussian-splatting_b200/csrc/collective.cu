// In-place all-reduce (sum) of the flat gradient bucket over NVLink SHARP (NVLS multimem).
//
// The path's only exchange step (SURVEY.md §8e) is the sum of the 134 MB gradient bucket that
// fused_project_bwd_kernel writes.  When that bucket lives in symmetric memory with a multicast
// mapping (torch.distributed._symmetric_memory), every rank reduces ONE 1/W slice of it with
// `multimem.ld_reduce` (the NVSwitch adds the W copies in flight) and writes the sum back to all W
// copies with `multimem.st` (the switch multicasts it): per GPU 134 MB out + 150 MB in instead of
// the 2 x 117 MB each way of a ring, and no staging copies.  Cross-rank ordering (all buckets
// written before / all slices broadcast after) is provided by the caller's symmetric-memory
// barriers; this kernel contains no spin loops.
#include <cstdlib>

#include "internal.h"

namespace {

__global__ void __launch_bounds__(512) nvls_allreduce_kernel(float4* __restrict__ mc, long long begin4,
                                                              long long end4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = begin4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end4; i += stride) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(mc + i)
                 : "memory");
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc + i), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
  }
}

// Two-shot all-reduce over plain peer (P2P) mappings: rank r sums slice r of all W copies with
// system-scope loads over NVLink and stores the sum into all W copies.  (W-1)/W * 2 bucket-sizes
// per direction - less than the multimem path for W = 2 (which moves 1 + 1/W), more for W >= 4.
// One owner per slice and a fixed summation order: every rank ends with the same bits.
struct GsPeers {
  float4* p[GS_MAX_PEERS];
};

__device__ __forceinline__ float4 ld_sys(const float4* a) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(a)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_sys(float4* a, float4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

template <int W>
__global__ void __launch_bounds__(512) p2p_allreduce_kernel(GsPeers peers, long long begin4, long long end4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = begin4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end4; i += stride) {
    float4 v[W];
#pragma unroll
    for (int p = 0; p < W; ++p) v[p] = ld_sys(peers.p[p] + i);
    float4 acc = v[0];
#pragma unroll
    for (int p = 1; p < W; ++p) {
      acc.x += v[p].x;
      acc.y += v[p].y;
      acc.z += v[p].z;
      acc.w += v[p].w;
    }
#pragma unroll
    for (int p = 0; p < W; ++p) st_sys(peers.p[p] + i, acc);
  }
}

// Second half of the pushed exchange (gs_grad_push): the owner of a slice sums its own bucket
// slice with the W-1 contributions its peers stored into its staging slots during THEIR projection
// backward (local HBM reads only) and stores the sum into all W buckets over NVLink.
template <int W>
__global__ void __launch_bounds__(512) push_finish_kernel(GsPeers buckets, const float4* own /* == buckets.p[rank]: no restrict */,
                                                          const float4* __restrict__ staging, long long per4,
                                                          int rank, long long begin4, long long end4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = begin4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end4; i += stride) {
    const long long j = i - begin4;
    float4 v[W];
#pragma unroll
    for (int p = 0; p < W; ++p) v[p] = p == rank ? own[i] : ld_sys(staging + p * per4 + j);
    float4 acc = v[0];
#pragma unroll
    for (int p = 1; p < W; ++p) {
      acc.x += v[p].x;
      acc.y += v[p].y;
      acc.z += v[p].z;
      acc.w += v[p].w;
    }
#pragma unroll
    for (int p = 0; p < W; ++p) st_sys(buckets.p[p] + i, acc);
  }
}

// Same second half with the broadcast done by the NVSwitch: ONE multimem.st per 16 bytes delivers the sum
// to all W buckets (each GPU sends its slice once instead of W-1 times; receive traffic is unchanged).
template <int W>
__global__ void __launch_bounds__(512) push_finish_mc_kernel(float4* mc_bucket, const float4* own,
                                                             const float4* __restrict__ staging, long long per4,
                                                             int rank, long long begin4, long long end4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = begin4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < end4; i += stride) {
    const long long j = i - begin4;
    float4 v[W];
#pragma unroll
    for (int p = 0; p < W; ++p) v[p] = p == rank ? own[i] : ld_sys(staging + p * per4 + j);
    float4 acc = v[0];
#pragma unroll
    for (int p = 1; p < W; ++p) {
      acc.x += v[p].x;
      acc.y += v[p].y;
      acc.z += v[p].z;
      acc.w += v[p].w;
    }
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_bucket + i), "f"(acc.x),
                 "f"(acc.y), "f"(acc.z), "f"(acc.w)
                 : "memory");
  }
}

int nvls_max_grid() {
  static const int g = [] {
    const char* e = getenv("GS_NVLS_GRID");          // tuning knob (CTAs), default 4 per SM of the current device
    if (e && atoi(e) > 0) return atoi(e);
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        sms <= 0)
      sms = 132;                                     // H100 SXM
    return sms * 4;
  }();
  return g;
}

}  // namespace

extern "C" int gs_allreduce_p2p_f32(void* const* peer_ptrs, long long n_floats, int rank, int world,
                                    gs_stream_t stream) {
  if (!peer_ptrs || n_floats < 0 || (n_floats % 4) || rank < 0 || rank >= world ||
      !(world == 2 || world == 4 || world == 8))
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_p2p_f32: bad arguments (world must be 2, 4 or 8)");
  GsPeers peers{};
  for (int p = 0; p < world; ++p) {
    if (!peer_ptrs[p] || reinterpret_cast<uintptr_t>(peer_ptrs[p]) % 16)
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_p2p_f32: peer pointers must be 16-byte aligned");
    peers.p[p] = static_cast<float4*>(peer_ptrs[p]);
  }
  const long long n4 = n_floats / 4;
  const long long per = (n4 + world - 1) / world;
  const long long begin4 = per * rank;
  const long long end4 = begin4 + per < n4 ? begin4 + per : n4;
  if (end4 <= begin4) return 0;
  int grid = (int)((end4 - begin4 + 511) / 512);
  if (grid > nvls_max_grid()) grid = nvls_max_grid();
  cudaStream_t st = (cudaStream_t)stream;
  if (world == 2) p2p_allreduce_kernel<2><<<grid, 512, 0, st>>>(peers, begin4, end4);
  else if (world == 4) p2p_allreduce_kernel<4><<<grid, 512, 0, st>>>(peers, begin4, end4);
  else p2p_allreduce_kernel<8><<<grid, 512, 0, st>>>(peers, begin4, end4);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_allreduce_push_finish_f32(void* const* peer_buckets, const float* staging_local, long long n_floats,
                                            long long per, int rank, int world, gs_stream_t stream) {
  if (!peer_buckets || !staging_local || n_floats < 0 || (n_floats % 4) || per <= 0 || (per % 4) || rank < 0 ||
      rank >= world || !(world == 2 || world == 4 || world == 8) || per * world < n_floats ||
      reinterpret_cast<uintptr_t>(staging_local) % 16)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_push_finish_f32: bad arguments");
  GsPeers peers{};
  for (int p = 0; p < world; ++p) {
    if (!peer_buckets[p] || reinterpret_cast<uintptr_t>(peer_buckets[p]) % 16)
      return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_push_finish_f32: bucket pointers must be 16-byte aligned");
    peers.p[p] = static_cast<float4*>(peer_buckets[p]);
  }
  const long long n4 = n_floats / 4, per4 = per / 4;
  const long long begin4 = per4 * rank;
  const long long end4 = begin4 + per4 < n4 ? begin4 + per4 : n4;
  if (end4 <= begin4) return 0;
  int grid = (int)((end4 - begin4 + 511) / 512);
  if (grid > nvls_max_grid()) grid = nvls_max_grid();
  cudaStream_t st = (cudaStream_t)stream;
  const float4* sg = reinterpret_cast<const float4*>(staging_local);
  if (world == 2) push_finish_kernel<2><<<grid, 512, 0, st>>>(peers, peers.p[rank], sg, per4, rank, begin4, end4);
  else if (world == 4) push_finish_kernel<4><<<grid, 512, 0, st>>>(peers, peers.p[rank], sg, per4, rank, begin4, end4);
  else push_finish_kernel<8><<<grid, 512, 0, st>>>(peers, peers.p[rank], sg, per4, rank, begin4, end4);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_allreduce_push_finish_mc_f32(void* bucket_multicast, const float* bucket_local,
                                               const float* staging_local, long long n_floats, long long per, int rank,
                                               int world, gs_stream_t stream) {
  if (!bucket_multicast || !bucket_local || !staging_local || n_floats < 0 || (n_floats % 4) || per <= 0 || (per % 4) ||
      rank < 0 || rank >= world || !(world == 2 || world == 4 || world == 8) || per * world < n_floats ||
      reinterpret_cast<uintptr_t>(staging_local) % 16 || reinterpret_cast<uintptr_t>(bucket_local) % 16 ||
      reinterpret_cast<uintptr_t>(bucket_multicast) % 16)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_push_finish_mc_f32: bad arguments");
  const long long n4 = n_floats / 4, per4 = per / 4;
  const long long begin4 = per4 * rank;
  const long long end4 = begin4 + per4 < n4 ? begin4 + per4 : n4;
  if (end4 <= begin4) return 0;
  int grid = (int)((end4 - begin4 + 511) / 512);
  if (grid > nvls_max_grid()) grid = nvls_max_grid();
  cudaStream_t st = (cudaStream_t)stream;
  float4* mc = static_cast<float4*>(bucket_multicast);
  const float4* own = reinterpret_cast<const float4*>(bucket_local);
  const float4* sg = reinterpret_cast<const float4*>(staging_local);
  if (world == 2) push_finish_mc_kernel<2><<<grid, 512, 0, st>>>(mc, own, sg, per4, rank, begin4, end4);
  else if (world == 4) push_finish_mc_kernel<4><<<grid, 512, 0, st>>>(mc, own, sg, per4, rank, begin4, end4);
  else push_finish_mc_kernel<8><<<grid, 512, 0, st>>>(mc, own, sg, per4, rank, begin4, end4);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}

extern "C" int gs_allreduce_multimem_f32(void* multicast_ptr, long long n_floats, int rank, int world,
                                         gs_stream_t stream) {
  if (!multicast_ptr || n_floats < 0 || (n_floats % 4) || world < 1 || rank < 0 || rank >= world)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_multimem_f32: bad arguments");
  if (reinterpret_cast<uintptr_t>(multicast_ptr) % 16)
    return gs_set_error_msg(GS_ERR_INVALID_ARG, "gs_allreduce_multimem_f32: pointer must be 16-byte aligned");
  const long long n4 = n_floats / 4;
  const long long per = (n4 + world - 1) / world;
  const long long begin4 = per * rank;
  const long long end4 = begin4 + per < n4 ? begin4 + per : n4;
  if (end4 <= begin4) return 0;
  const long long work = end4 - begin4;
  int grid = (int)((work + 511) / 512);
  if (grid > nvls_max_grid()) grid = nvls_max_grid();
  nvls_allreduce_kernel<<<grid, 512, 0, (cudaStream_t)stream>>>(static_cast<float4*>(multicast_ptr), begin4, end4);
  GS_CUDA_TRY(cudaGetLastError());
  gs_count_launch();
  return 0;
}
