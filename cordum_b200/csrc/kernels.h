// kernels.h — kernel parameter block and launchers (kernels.cu <-> engine.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/cordum_b200.h"
#include "tables.h"

struct KParams {
  JobRecords recs;        // device pointers to the encoded (topic-sorted) records of this batch
  DeviceTables t;         // device pointers to the compiled tables
  cordum_decision* out;   // device, n_jobs records
  uint32_t n_jobs;
  uint32_t* route_count;     // device: number of jobs policy_kernel found dispatchable (null: no compaction)
  uint2* route_list;         // device: {slot in the sorted records, head word policy_kernel wrote} per dispatchable job
  uint32_t honor_approved;   // POLICY_AND_ROUTE: jobs flagged JF_APPROVED bypass the policy (engine.go:484-522)
};

// peer-memory heartbeat exchange (kernels.cu peer_push_kernel)
#define CORDUM_MAX_PEERS 16
struct PeerPush {
  uint32_t rank, world, per;                 // per = worker slots per rank
  const uint32_t* epoch_ptr;                 // device: the epoch this launch announces and waits for (copied in with the slice)
  const Load16* my_slice;                    // local: this rank's slice inside its own table of this epoch's parity
  Load16* peer_slices[CORDUM_MAX_PEERS];     // where this rank's slice goes in every peer's table of that parity
  uint32_t* peer_flags[CORDUM_MAX_PEERS];    // every rank's flag array [CORDUM_MAX_PEERS]: peer_flags[q][r] = last epoch rank r announced to q
  const uint32_t* my_flags;                  // = peer_flags[rank]
  uint32_t* done_ctr;                        // local scratch: CTAs that have finished pushing
};
cudaError_t launch_peer_push(const PeerPush& G, cudaStream_t s);
cudaError_t launch_configure();

// loads_read (optional) is recorded once T.loads has been consumed (between the chunk and the merge kernel)
cudaError_t launch_worker_pools(const DeviceTables& T, cudaStream_t s, cudaEvent_t loads_read);   // chunk sort, merge, label_best
cudaError_t launch_policy(const KParams& P, int sm_count, cudaStream_t s, int share = 0);
// route_kernel, then route_select_kernel when the tables hold selective pairs and the batch lists jobs that name them
cudaError_t launch_route(const KParams& P, bool route_only, int sm_count, cudaStream_t s, int share = 0);
inline uint32_t route_launches(const KParams& P) { return P.n_jobs ? 1u + (P.t.n_sel && P.recs.n_sel_jobs ? 1u : 0u) : 0u; }

// ---- device-side encoder (encode.cu)
struct EncodeParams {
  uint32_t n_jobs;
  EncodeTables et;                 // device pointers (the engine rebases Host::export_dicts' offsets)
  // the envelope arrays of include/cordum_b200.h cordum_envelopes, on the device
  const uint8_t* arena;
  const cordum_str *topic, *tenant, *principal_id, *effective_config, *meta_tenant_id, *actor_id, *capability, *pack_id;
  const uint8_t *has_meta, *actor_type, *approved;
  const uint32_t *risk_off, *requires_off, *label_off;
  const cordum_str *risk_tags, *requires_, *label_keys, *label_vals;
  // work arrays (device)
  uint32_t *tid, *ten, *key, *hist, *slot_of, *fallback;
  JobRec* out_job;
  RouteRec* out_route;
};
cudaError_t launch_encode(const EncodeParams& P, uint32_t n_keys, cudaStream_t s);
