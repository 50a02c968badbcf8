// sync.cu — one-shot all-reduce of small per-layer vectors over NVLink peer memory, for synchronised BatchNorm
// (SURVEY.md 8e collective (2), 5.8: "all-reduce [sum x, sum x^2] per BN in forward and [sum dy, sum dy xhat] in
// backward, fp32, low-latency").  A BatchNorm needs 2C floats (512 B .. 16 KB) from every rank between the conv that
// produces them and the normalisation pass that consumes them: pure latency.  NCCL spends 10-20 us per such call.  Here
// every rank owns a RECEIVE buffer [world][sum 2C] of (value, stamp) pairs in symmetric memory (mapped into every peer by
// torch's symmetric-memory rendezvous -- plumbing), and one small CTA per rank
//   1. PUSHES its partial sums, each paired with the current step stamp in ONE 8-byte store, into slot [my rank] of every
//      peer's receive buffer (posted NVLink stores: one-way latency, no request / response round trip, and -- because
//      the stamp travels inside the same atomic 8-byte word as the value -- no system-scope fence and no separate flag),
//   2. polls its OWN receive slots until every pair carries this step's stamp (local memory),
//   3. adds the world contributions IN RANK ORDER (its own partial sums + the received values), so every rank computes
//      bit-identical totals and the replicas stay identical.
// The partial sums are complete when the kernel starts (stream order behind their producer).  Reuse across steps is
// safe because a peer can push the next step's values of an exchange only after the gradient all-reduce of this step,
// which every rank joins after its last exchange.  The step stamp lives in device memory (bumped by a tiny kernel at
// the start of every forward), so the launches replay unchanged inside CUDA graphs.
#include "host_common.h"
#include "sync.cuh"
#include "../../include/mcb200.h"

namespace mcb {

__global__ void sync_step_bump_kernel(unsigned* step) {
  if (threadIdx.x == 0) *step = *step + 1u;
}

constexpr int kSyncThreads = 1024;
__global__ void __launch_bounds__(kSyncThreads) sync_exchange_kernel(SyncDesc d) { sync_exchange_block(d); }

}  // namespace mcb

using namespace mcb;

extern "C" int mcb_sync_step_bump(unsigned* step, void* stream) {
  MCB_REQUIRE(step, "sync_step_bump: null pointer");
  sync_step_bump_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(step);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}

extern "C" int mcb_sync_exchange(const float* partial, void* const* peer_recv, int rank, int world, long stride, long offset,
                                 int count, const unsigned* step, float* out, float* out2_first, float* out2_second,
                                 int split, float scale2, void* stream) {
  MCB_REQUIRE(partial && peer_recv && step && out, "sync_exchange: null pointer");
  MCB_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world && count > 0, "sync_exchange: bad rank / world / count");
  MCB_REQUIRE((out2_first == nullptr) == (out2_second == nullptr) && split >= 0 && split <= count, "sync_exchange: bad split");
  SyncDesc d{partial, reinterpret_cast<float2* const*>(peer_recv), rank, world, stride, offset, count, step, out, out2_first,
             out2_second, split, scale2};
  sync_exchange_kernel<<<1, kSyncThreads, 0, static_cast<cudaStream_t>(stream)>>>(d);
  MCB_LAUNCH_CHECK();
  return MCB_OK;
}
