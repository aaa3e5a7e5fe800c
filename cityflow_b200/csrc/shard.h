// Multi-GPU execution of one simulation: one process per GPU, the road graph cut by intersection
// (partition.h), the seam records exchanged on the engine's CUDA stream.
//
// Per step and rank (DeviceSim::shardStep; DeviceSim::shardSegment runs the same sequence in three pieces, cut at
// X1 and X2, for a caller that moves the records itself):
//   stage + k_ingest                       admission into owned lanes -- and, identically, into the ghost
//                                          copies of the lanes this rank feeds (so no exchange is needed here)
//   k_notify, k_control
//   X1  movers     feeder -> owner         vehicles that left a laneLink into a seam lane
//   k_move
//   X2  tails      owner -> feeder         + every rank's blocker changes to every rank, one NCCL group
//   k_leader
// Host bookkeeping (RNG, flows, ids) is replicated: every rank runs the same spawner and ingests
// only the records of lanes it owns; finished vehicles are all-gathered when the host drains.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "device_sim.h"

namespace cfb {

class ShardTransport {
public:
    virtual ~ShardTransport() {}
    virtual int rank() const = 0;
    virtual int world() const = 0;
    // send[beg_s[q]..beg_s[q+1]) -> peer q; recv[beg_r[q]..beg_r[q+1]) <- peer q; entries of `bytes`
    virtual void exchange(void *stream, const void *send, const std::vector<int> &sendBeg, void *recv,
                          const std::vector<int> &recvBeg, size_t bytes) = 0;
    virtual void allGather(void *stream, const void *send, void *recvAll, size_t bytesPerRank) = 0;
    // exchange() and allGather() issued as ONE group (one launch on the stream)
    virtual void exchangeAndGather(void *stream, const void *send, const std::vector<int> &sendBeg, void *recv,
                                   const std::vector<int> &recvBeg, size_t bytes, const void *gSend, void *gRecvAll,
                                   size_t gBytesPerRank) = 0;
    virtual void allReduceSumInt(void *stream, int *devBuf, int n) = 0;   // in place, device ints
    // Peer-memory data plane (device_shard.cuh): make `localBase` (one cudaMalloc of `bytes`) writable by every other
    // rank and map theirs.  peerBase[q] = rank q's arena in this process's address space (own entry = localBase).
    // Returns false (with `err`) when some pair of GPUs cannot reach each other; every rank gets the same answer.
    virtual bool shareArena(void *localBase, size_t bytes, std::vector<void *> &peerBase, std::string &err) = 0;
};

// NCCL transport (libnccl is loaded at run time with dlopen, so the single-GPU engine has no
// dependency on it).  `uniqueId` = the 128-byte ncclUniqueId created by rank 0.
ShardTransport *createNcclTransport(int rank, int world, const void *uniqueId, int device, std::string &err);
// 128-byte id for createNcclTransport (call on one rank, broadcast by any means)
bool ncclUniqueIdBytes(unsigned char out[128], std::string &err);

}  // namespace cfb
