// What the multi-GPU drivers share: the pnr_mgpu handle (csrc/pnr_mgpu.cu creates it), the torch.chunk shard bounds
// and the per-shard streams.  Included by pnr_mgpu.cu (render, backward) and pnr_mgpu_field.cu (field evaluation).
#pragma once
#include <stdint.h>

#include <vector>

#include "pnr_common.cuh"

#define PNR_MGPU_MAX_SOURCES 63   // pnr_mgpu_create takes at most 64 devices: device 0 plus 63 sources

struct PnrMgpu {
  std::vector<int> dev;
  std::vector<cudaStream_t> stream;   // per device (index 0 unused: device 0 work runs on the caller's stream)
  std::vector<cudaEvent_t> done;      // per device
  std::vector<char> peer_to_0;        // device i can address device 0's memory
  std::vector<char> peer_from_0;      // device 0 can address device i's memory (the backward's reduction reads it)
  cudaEvent_t start;                  // recorded on the caller's stream of device 0
  cudaEvent_t reduced;                // recorded on device 0 after the backward's reduction
};

namespace pnr {

struct DevGuard {
  int prev;
  DevGuard() { cudaGetDevice(&prev); }
  ~DevGuard() { cudaSetDevice(prev); }
};

// torch.chunk piece i of n over B rays: [a, b)
static void chunk_bounds(int64_t B, int n, int i, int64_t* a, int64_t* b) {
  const int64_t per = (B + n - 1) / n;
  *a = per * i < B ? per * i : B;
  *b = *a + per < B ? *a + per : B;
}

// The stream each shard is enqueued on: shard 0 uses the caller's stream, shard i its requested stream (NULL: the
// handle's own) -- except that shards on the same device all take the stream of the first shard there.  The tensor
// engine's fused render kernel spins on flags set by other CTAs of the same launch (DESIGN.md 3.1), which is deadlock
// free only while the whole persistent grid is resident; two such launches running at once on one GPU break that.
template <class Requested>
static std::vector<cudaStream_t> shard_streams(const PnrMgpu* h, cudaStream_t stream0, Requested requested) {
  const int n = (int)h->dev.size();
  std::vector<cudaStream_t> s(n);
  for (int i = 0; i < n; ++i) {
    s[i] = i == 0 ? stream0 : (requested(i) ? (cudaStream_t)requested(i) : h->stream[i]);
    for (int j = 0; j < i; ++j)
      if (h->dev[j] == h->dev[i]) {
        s[i] = s[j];
        break;
      }
  }
  return s;
}


}  // namespace pnr
