// device_shard.cuh -- what crosses a seam of a sharded run (partition.h, shard.h): the seam records, and the protocol
// that moves them over PEER MEMORY (NVLink / NVSwitch) or, staged, through a ShardTransport.
// Part of device_sim.cu.  The reference has no counterpart (its threads share one address space).
//
// Every rank owns one "arena" (one cudaMalloc, exported with cudaIpc and mapped by every peer):
//
//   flags   [3][world] int    flags[k][src] = last epoch for which rank `src` completed its writes of kind k
//                              k = 0 movers of the step, 1 tails + blocker list of the step, 2 finished-vehicle marks
//           [8][world] int    activeOf[E % 8][src] = rank `src`'s share of get_vehicle_count() after step E (every rank
//                              stores it into every arena: the collective count needs no all-reduce, k_sum_active)
//   delStep [slotCap]   int   step at which the vehicle of a slot left the network (every rank writes here)
//   blkIn   [2][world][1 + BLK_IN_CAP] int2   this step's blocker changes of a NEIGHBOUR rank, count in [0].x
//   moverIn [2][nBoundIn]  MoverMsg            entrants of the lanes this rank owns and a peer feeds
//   tailIn  [2][nBoundOut] TailMsg             tail records of the lanes this rank feeds and a peer owns
//
// A sender stores its records straight into the receiver's arena (posted writes over NVLink), fences, and the
// last block of the sending kernel publishes the epoch in the receiver's flag word; the receiving kernel spins on
// its LOCAL flag word and then reads its LOCAL mailbox.  No collective, no host involvement, two dependent
// NVLink hops per step (movers after k_control, tails after k_move).  The [2] is the parity of the epoch: a
// sender can be at most one step ahead of a neighbour that still reads the previous message (shard.h).
//
// Deadlock freedom: a kernel only ever waits for data whose producing kernel depends on nothing later than what the
// waiting rank has already sent (movers(t) <- k_control(t) <- tails(t-1) <- k_move(t-1) <- movers(t-1) ...).  Every wait
// has a time-out (ERR_SHARD_TIMEOUT) so a crashed peer cannot hang the GPU.
#pragma once

namespace cfb {

constexpr int BLK_IN_CAP = 1 << 13;     // blocker changes per step sent to one neighbour (8 bytes each)
constexpr int SHARD_ACT_RING = 8;       // per-step vehicle counts of the other ranks: a ring deeper than any rank can run ahead
constexpr int SHARD_FLAG_KINDS = 3 + SHARD_ACT_RING;   // flag words 0..2, then activeOf[E % ring][src]
constexpr long long SHARD_SPIN_LIMIT_NS = 4000000000LL;   // 4 s

struct __align__(16) TailMsg {     // owner -> feeder: Drivable::getLastVehicle of a boundary lane
    Tail tail;
    int count, inserted, pad0, pad1;
    double2 kin;
    int4 ids, nav;
};
struct __align__(16) MoverRec {
    double2 kin;
    int4 ids, nav;
};
struct __align__(16) MoverMsg {    // feeder -> owner: this step's entrants of a boundary lane
    int n, pad0, pad1, pad2;
    MoverRec rec[ENT_CAP];
};

struct ShardPeer {                 // rank q's arena as mapped into this process (all null for q == me)
    int *flags;
    int *delStep;
    int2 *blkIn;                   // q's blkIn[0][me]; parity 1 is `blkStride` further
    MoverMsg *moverIn;             // q's moverIn[0]; parity 1 is nIn further
    TailMsg *tailIn;
    int nIn, nOut;                 // q's nBoundIn / nBoundOut (strides of the parity halves)
};

struct ShardP2P {                  // by-value kernel argument
    const ShardPeer *peers;        // [world]
    int me, world;
    const int *nbr;                // ranks that share a seam lane with me
    int nNbr;
    const int *outPeer, *outDst;   // per boundOut entry: owner rank, index in the owner's moverIn
    const int *inPeer, *inDst;     // per boundIn entry: feeder rank, index in the feeder's tailIn
    int *flags;                    // my own arena
    int2 *blkIn;
    MoverMsg *moverIn;
    TailMsg *tailIn;
    int *ticket;                   // 2 ints: block tickets of the two sending kernels
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long shardNow() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void shardPause() { __nanosleep(100); }
#else   // tests/device_sim_emu.cpp runs these bodies on the host: every poll counts as a millisecond, so a flag that never
        // comes (a protocol error) trips the time-out instead of spinning for ever
static unsigned long long g_shardClock = 0;
inline unsigned long long shardNow() { return g_shardClock += 1000000ULL; }
inline void shardPause() {}
#endif

// Block-wide: wait until every neighbour's flag of `kind` has reached epoch E.
__device__ __forceinline__ void shardWait(const View &V, const ShardP2P &S, int kind, int E, bool allRanks) {
    if (threadIdx.x == 0) {
        const unsigned long long t0 = shardNow();
        const int n = allRanks ? S.world : S.nNbr;
        for (int k = 0; k < n; ++k) {
            const int q = allRanks ? k : S.nbr[k];
            if (q == S.me) continue;
            volatile int *f = S.flags + kind * S.world + q;
            while (*f < E) {
                if (shardNow() - t0 > (unsigned long long) SHARD_SPIN_LIMIT_NS) {
                    atomicOr(&V.ctrl->error, ERR_SHARD_TIMEOUT);
                    break;
                }
                shardPause();
            }
        }
        __threadfence_system();   // acquire: the mailbox reads below come after the flag reads
    }
    __syncthreads();
}

// Called by every thread after its remote stores: the last block to arrive publishes the epoch.  Ordering: every
// thread's stores -> the block barrier -> ONE system-scope fence per block by thread 0 (fences are cumulative: it orders
// everything that happened before it, for every observer in the system) -> the ticket (device-scope atomic) -> observed
// by the last block -> its fence -> the flag.  (A system-scope fence in EVERY thread cost several microseconds per send
// kernel, r02d: each waits for the NVLink acknowledgement of the stores before it.)
__device__ __forceinline__ bool shardLastBlock(int *ticket) {
    __shared__ int sLast;
    __syncthreads();                  // the block's stores happen before thread 0's fence (CTA barrier) ...
    if (threadIdx.x == 0) {
        __threadfence_system();       // ... which is cumulative: one fence per block covers all of them
        const int t = atomicAdd(ticket, 1);
        sLast = (t == (int) gridDim.x - 1);
        if (sLast) {
            *ticket = 0;
            __threadfence_system();   // acquire side of the ticket: every block's fence is ordered before the flag stores
        }
    }
    __syncthreads();
    return sLast != 0;
}
// programmatic dependent launch (see pdlEnter() in device_sim.cu)
__device__ __forceinline__ void shardPdlEnter() {
#ifdef __CUDACC__
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}

// ---- the seam records, one definition each: the peer-memory bodies below and the staged kernels (k_pack_* / k_unpack_*)
// differ only in where a record is stored and where it is read from ----

// Owner side: the tail record of boundary lane L (Drivable::getLastVehicle) with the state of that vehicle.
__device__ __forceinline__ TailMsg tailMsgOf(const View &V, int L) {
    TailMsg m;
    m.tail = V.tail[L];
    m.count = V.count[L];
    m.inserted = V.inserted[L];
    m.pad0 = m.pad1 = 0;
    m.kin = make_double2(0, 0);
    m.ids = m.nav = make_int4(0, 0, 0, 0);
    if (m.tail.pos >= 0) {
        m.kin = V.kin[m.tail.pos];
        m.ids = V.ids[m.tail.pos];
        m.nav = V.nav[m.tail.pos];
    }
    return m;
}
// Feeder side: refresh boundary lane L from its owner's tail record.
__device__ __forceinline__ void applyTailMsg(const View &V, int L, const TailMsg m) {   // (a copy: every load before the stores)
    V.tail[L] = m.tail;
    V.count[L] = m.count;
    V.inserted[L] = (unsigned char) m.inserted;
    if (m.tail.pos >= 0) {  // ghost copy of the one vehicle this rank may look at
        V.kin[m.tail.pos] = m.kin;
        V.ids[m.tail.pos] = m.ids;
        V.nav[m.tail.pos] = m.nav;
    }
}
// Feeder side, one warp per lane: this step's entrants of boundary lane L into `out`; they leave this rank.
__device__ __forceinline__ void fillMoverMsg(const View &V, int L, MoverMsg *out, int lane) {
    const int n = min(V.entCnt[L], ENT_CAP);
    if (lane == 0) { out->n = n; out->pad0 = out->pad1 = out->pad2 = 0; }
    if (lane < n) {
        const int m = V.ent[L * ENT_CAP + lane];
        MoverRec r;
        r.kin = V.mkin[m];
        r.ids = V.mids[m];
        r.nav = V.mnav[m];
        out->rec[lane] = r;
    }
    __syncwarp();
    if (lane == 0) V.entCnt[L] = 0;
}
// Owner side, one warp per lane: stage the entrants of boundary lane L like local movers.
__device__ __forceinline__ void stageMoverMsg(const View &V, int L, const MoverMsg *in, int lane) {
    const int n = in->n;
    if (n == 0) return;
    int base = 0;
    if (lane == 0) base = atomicAdd(&V.ctrl->moverCount, n);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (lane < n) {
        const int m = base + lane;
        if (m < V.moverCap) {
            const MoverRec r = in->rec[lane];
            V.mkin[m] = r.kin;
            V.mids[m] = r.ids;
            V.mnav[m] = r.nav;
            V.ent[L * ENT_CAP + lane] = m;
        } else {
            atomicOr(&V.ctrl->error, ERR_MOVER_OVERFLOW);
        }
    }
    if (lane == 0) {
        V.entCnt[L] = n;
        if (V.count[L] == 0) V.extraList[atomicAdd(&V.ctrl->nExtra, 1)] = L;
    }
}
// One blocker change of another rank: u = (slot, blocker slot), blocker -2 = the vehicle left the network at `step`.
__device__ __forceinline__ void applyBlkChange(const View &V, int2 u, int step) {
    if (u.y == -2) {
        V.blk[u.x] = -1;
        V.delStep[u.x] = step;
    } else {
        V.blk[u.x] = u.y;
    }
}

// After k_control: one warp per boundary lane this rank feeds; the record goes straight into the owner's arena.
__device__ __forceinline__ void sendMoversBody(const View &V, const ShardP2P &S) {
    const int E = V.ctrl->epoch + 1, par = E & 1;
    const int nW = (gridDim.x * blockDim.x) >> 5;
    for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < V.nBoundOut; j += nW) {
        const ShardPeer &P = S.peers[S.outPeer[j]];
        fillMoverMsg(V, V.boundOut[j], P.moverIn + (size_t) par * P.nIn + S.outDst[j], threadIdx.x & 31);
    }
    if (shardLastBlock(S.ticket) && threadIdx.x == 0)   // (the thread that issued the system fence)
        for (int k = 0; k < S.nNbr; ++k) *(volatile int *) (S.peers[S.nbr[k]].flags + 0 * S.world + S.me) = E;
}
__global__ void __launch_bounds__(128) k_send_movers(View V, ShardP2P S) { shardPdlEnter(); sendMoversBody(V, S); }

// Before k_move: wait for the feeders, then stage their entrants like local movers.
__device__ __forceinline__ void recvMoversBody(const View &V, const ShardP2P &S) {
    const int E = V.ctrl->epoch + 1, par = E & 1;
    shardWait(V, S, 0, E, false);
    const int nW = (gridDim.x * blockDim.x) >> 5;
    const MoverMsg *in = S.moverIn + (size_t) par * V.nBoundIn;
    for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < V.nBoundIn; j += nW)
        stageMoverMsg(V, V.boundIn[j], in + j, threadIdx.x & 31);
}
__global__ void __launch_bounds__(128) k_recv_movers(View V, ShardP2P S) { shardPdlEnter(); recvMoversBody(V, S); }
// Both halves in one launch (the default): this rank's sends do not depend on what it receives, so the kernel first
// stores and publishes its own records and then waits for the neighbours' -- one launch and one ramp less per exchange.
__global__ void __launch_bounds__(128) k_xchg_movers(View V, ShardP2P S) { shardPdlEnter(); sendMoversBody(V, S); recvMoversBody(V, S); }

// After k_move: tail records to the feeders, this step's blocker changes to the neighbours, finished-vehicle marks
// to everybody.
__device__ __forceinline__ void sendTailsBody(const View &V, const ShardP2P &S) {
    const int E = V.ctrl->epoch + 1, par = E & 1;
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    for (int j = gtid; j < V.nBoundIn; j += stride) {
        const ShardPeer &P = S.peers[S.inPeer[j]];
        P.tailIn[(size_t) par * P.nOut + S.inDst[j]] = tailMsgOf(V, V.boundIn[j]);
    }
    const int nUpd = V.ctrl->nBlkUpd;
    if (nUpd > BLK_IN_CAP) atomicOr(&V.ctrl->error, ERR_MOVER_OVERFLOW);
    const int n = min(nUpd, BLK_IN_CAP);
    const size_t blkStride = (size_t) S.world * (1 + BLK_IN_CAP);
    for (int k = 0; k < S.nNbr; ++k) {
        int2 *dst = S.peers[S.nbr[k]].blkIn + (size_t) par * blkStride;
        for (int i = gtid; i < n; i += stride) dst[1 + i] = V.blkUpd[1 + i];
        if (gtid == 0) dst[0] = make_int2(n, E);
    }
    const int step = V.ctrl->step;
    for (int i = gtid; i < n; i += stride) {
        const int2 u = V.blkUpd[1 + i];
        if (u.y != -2) continue;
        for (int q = 0; q < S.world; ++q)
            if (q != S.me) S.peers[q].delStep[u.x] = step;
    }
    if (shardLastBlock(S.ticket + 1) && threadIdx.x == 0) {   // (the thread that issued the system fence)
        V.ctrl->nBlkUpd = 0;
        for (int k = 0; k < S.nNbr; ++k) *(volatile int *) (S.peers[S.nbr[k]].flags + 1 * S.world + S.me) = E;   // (what the neighbours wait for goes first)
        const int act = V.ctrl->active;                        // final for this step: k_move is done
        for (int q = 0; q < S.world; ++q)
            if (q != S.me) *(volatile int *) (S.peers[q].flags + (3 + E % SHARD_ACT_RING) * S.world + S.me) = act;
        __threadfence_system();
        for (int q = 0; q < S.world; ++q)
            if (q != S.me) *(volatile int *) (S.peers[q].flags + 2 * S.world + S.me) = E;
    }
}
__global__ void __launch_bounds__(128) k_send_tails(View V, ShardP2P S) { shardPdlEnter(); sendTailsBody(V, S); }

// Before k_leader: wait for the owners / neighbours, refresh the ghost copies, apply the neighbours' blocker changes.
__device__ __forceinline__ void recvTailsBody(const View &V, const ShardP2P &S) {
    const int E = V.ctrl->epoch + 1, par = E & 1;
    shardWait(V, S, 1, E, false);
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    const TailMsg *in = S.tailIn + (size_t) par * V.nBoundOut;
    for (int j = gtid; j < V.nBoundOut; j += stride) applyTailMsg(V, V.boundOut[j], in[j]);
    const size_t blkStride = (size_t) S.world * (1 + BLK_IN_CAP);
    const int step = V.ctrl->step;
    for (int k = 0; k < S.nNbr; ++k) {
        const int2 *src = S.blkIn + (size_t) par * blkStride + (size_t) S.nbr[k] * (1 + BLK_IN_CAP);
        const int n = src[0].x;
        for (int i = gtid; i < n; i += stride) applyBlkChange(V, src[1 + i], step);
    }
}
__global__ void __launch_bounds__(128) k_recv_tails(View V, ShardP2P S) { shardPdlEnter(); recvTailsBody(V, S); }
__global__ void __launch_bounds__(128) k_xchg_tails(View V, ShardP2P S) { shardPdlEnter(); sendTailsBody(V, S); recvTailsBody(V, S); }

// ---- the staged form: the same records through the engine's send / receive buffers, moved between the ranks by a
// ShardTransport (CITYFLOW_B200_SHARD_TRANSPORT=nccl) ----
__global__ void k_pack_tails(View V, TailMsg *out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < V.nBoundIn) out[j] = tailMsgOf(V, V.boundIn[j]);
}
__global__ void k_unpack_tails(View V, const TailMsg *in) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < V.nBoundOut) applyTailMsg(V, V.boundOut[j], in[j]);
}
__global__ void k_pack_movers(View V, MoverMsg *out) {  // one warp per boundary lane this rank feeds
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j < V.nBoundOut) fillMoverMsg(V, V.boundOut[j], out + j, threadIdx.x & 31);
}
__global__ void k_unpack_movers(View V, const MoverMsg *in) {  // one warp per boundary lane this rank owns
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j < V.nBoundIn) stageMoverMsg(V, V.boundIn[j], in + j, threadIdx.x & 31);
}
// blocker changes: [0] = {count,0} header, filled right before the all-gather
__global__ void k_seal_blk(View V) {
    V.blkUpd[0] = make_int2(min(V.ctrl->nBlkUpd, V.blkUpdCap), 0);
    V.ctrl->nBlkUpd = 0;
}
// every other rank's list, one rank per blockIdx.y
__global__ void k_apply_blk(View V, const int2 *all, int me, int stridePerRank) {
    const int r = blockIdx.y;
    if (r == me) return;
    const int2 *src = all + (size_t) r * stridePerRank;
    const int n = src[0].x, step = V.ctrl->step;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) applyBlkChange(V, src[1 + i], step);
}

// Host query support: every rank's finished-vehicle marks through the last completed step have landed here.
__global__ void k_wait_fin(View V, ShardP2P S) { shardWait(V, S, 2, V.ctrl->epoch, true); }

// The collective get_vehicle_count() (engine.cpp:615-617 over the whole network) without a collective: every rank's share
// of the last completed step is already in this arena; wait for the stamps, add them up, hand the sum to the host
// through its mapped mirror (words 4, 5 = sum, epoch).
__global__ void k_sum_active(View V, ShardP2P S) {
    const int E = V.ctrl->epoch;
    shardWait(V, S, 2, E, true);
    if (threadIdx.x == 0 && V.hostMirror) {
        long long sum = V.ctrl->active;
        for (int q = 0; q < S.world; ++q)
            if (q != S.me) sum += *(volatile int *) (S.flags + (3 + E % SHARD_ACT_RING) * S.world + q);
        volatile int *m = V.hostMirror;
        m[4] = (int) sum;
        m[6] = V.ctrl->error;
        __threadfence_system();
        m[5] = E;
    }
}

}  // namespace cfb
