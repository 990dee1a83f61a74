// raft_common.cuh -- device side of the batched multi-Raft engine (sm_90a): what both passes of the logic share
// (raft_step.cuh includes raft_logic.cuh / raft_row_logic.cuh twice: 64-bit and 32-bit index arithmetic).
//
// One thread owns one member row for the whole launch ("owner computes"): every HBM column
// is indexed by row, rows are slot-major (row = slot * n_groups + group), so the 32 lanes
// of a warp touch 32 consecutive 16-byte cells of each column -> one fully coalesced
// 512-byte request per column pair (LDG.E.128 / STG.E.128).  The Raft decision logic is
// integer compare/min/max/select; no tensor cores.
//
// What is evaluated (reference: rabbitmq/ra v3.1.6 src/ra_server.erl):
//   handle_leader/2    :520-1023   AER-reply (success / failure back-off / higher term),
//                                  command(s), written event, pipeline_rpcs, AER, votes
//   handle_follower/2  :1264-1641  AER (log match, truncate, write), written event, votes
//   handle_candidate/2 :1026-1171, handle_pre_vote/2 :1173-1261,
//   handle_await_condition/2 :1900-1941 + follower_catchup_cond/3 :2184-2213
//   evaluate_quorum/2 :3606-3619, agreed_commit/1 :3657-3661 (rank select, no sort),
//   make_pipelined_rpc_effects/3 :2268-2329, make_rpc_effect/5 :2365-2399,
//   call_for_election/3 :2853-2897, process_pre_vote/3 :2899-2956
// plus the slice of ra_server_proc that feeds back into it inside one mailbox turn
// ({next_event,_} chasing :1574-1577, become/3 via handle_state_enter, tick on election win).
//
// The log facade (src/ra_log.erl fetch_term/exists/write/set_last_index/handle_event
// {written}) is a run-length index->term view: at most RA_MAX_RUNS (start, term) runs per
// member, so no per-entry storage lives on the GPU.
#pragma once
#include <stdint.h>
#include "../../include/ra_engine.h"

typedef unsigned long long u64;
typedef long long i64;
typedef unsigned int u32;
typedef unsigned char u8;

#define RA_UNDEF 0xFFFFFFFFFFFFFFFFull

// ---- meta word (second half of the `ap` pair) -------------------------------------
//  [0:3) role  [3:7) leader  [7:11) voted_for  [11:13) membership  [13:15) condition
//  [15:19) votes  [19:23) n_runs  23 has_snapshot  24 pipeline_pending  25 cond_reply_valid
//  26 fatal  27 mv_ok  [28:32) idle  [32:56) peer status 3b x 8  [56:64) voter mask
#define MT_ROLE(m)        ((u32)((m) & 7ull))
#define MT_LEADER(m)      ((u32)(((m) >> 3) & 15ull))
#define MT_VOTED(m)       ((u32)(((m) >> 7) & 15ull))
#define MT_MEMBERSHIP(m)  ((u32)(((m) >> 11) & 3ull))
#define MT_COND(m)        ((u32)(((m) >> 13) & 3ull))
#define MT_VOTES(m)       ((u32)(((m) >> 15) & 15ull))
#define MT_NRUNS(m)       ((u32)(((m) >> 19) & 15ull))
#define MT_HAS_SNAP(m)    ((u32)(((m) >> 23) & 1ull))
#define MT_PIPE_PEND(m)   ((u32)(((m) >> 24) & 1ull))
#define MT_COND_VALID(m)  ((u32)(((m) >> 25) & 1ull))
#define MT_FATAL(m)       ((u32)(((m) >> 26) & 1ull))
#define MT_MV_OK(m)       ((u32)(((m) >> 27) & 1ull))
#define MT_IDLE(m)        ((u32)(((m) >> 28) & 15ull))
#define MT_PSTATUS(m, s)  ((u32)(((m) >> (32 + 3 * (s))) & 7ull))
#define MT_VOTER(m, s)    ((u32)(((m) >> (56 + (s))) & 1ull))
#define MT_SET(m, sh, w, v) ((m) = ((m) & ~((((u64)1 << (w)) - 1) << (sh))) | (((u64)(v) & (((u64)1 << (w)) - 1)) << (sh)))
#define SLOT_NONE 15u
// The template int of the device functions carries two compile-time specialisations:
//   low byte  = number of members (0: read it from the config)
//   next byte = transport of the RPC records (0: decide at run time)
// so that the hot kernel contains the code of exactly one transport (instruction-cache footprint).
#define TR_RUNTIME 0
#define TR_LOCAL   1   /* route_on_device, one shard: mailbox planes of this GPU          */
#define TR_PEER    2   /* n_shards > 1: NVLink peer stores into the destination GPU      */
#define TR_BUCKET  3   /* n_shards > 1: per-destination buckets for the all-to-all       */
#define TR_HOST    4   /* not routed: records returned to the host (omsg slots)          */
#define MK_MM(members, tr) ((members) | ((tr) << 8))
#define MMEM (MM & 0xff)
#define MTR  ((MM >> 8) & 0xff)
#define NMEM(C) ((u32)(MMEM ? MMEM : (C).members))
#define PSTR (MMEM ? MMEM : RA_MAX_MEMBERS)      // peer slots staged per thread in shared memory

struct Cols {
    // scalar pairs, one cell per row
    ulonglong2* tc;     // {current_term, commit_index}
    ulonglong2* lg;     // {last_index, last_term}
    ulonglong2* lw;     // {last_written_index, last_written_term}
    ulonglong2* ap;     // {last_applied, meta}
    ulonglong2* sn;     // {snapshot_index, snapshot_term}
    ulonglong2* tk;     // {pre_vote_token, token_counter}
    ulonglong2* fm;     // {first_index, machine_version | effective_machine_version << 32}
    ulonglong2* cd;     // [2][rows] await_condition reply {term,next},{last_index,last_term}
    // per peer slot s: [s][rows]
    ulonglong2* pnm;    // {next_index, match_index}
    u64*        pcs;    // commit_index_sent
    // log view: [k][rows] {run_start, run_term}
    ulonglong2* run;
    // consistent queries: own query_index, highest index the host was told a quorum agreed on, and per
    // peer slot s: [s][rows] the peer's query_index (ra_server_state() :96, ra_peer_state() ra.hrl:63-75)
    u64*        qi;
    u64*        qa;
    u64*        pqi;
    u64*        wc;     // [rows] compact note stream: term of the last WAL_APPEND note the host was told for this row
    u8*         wf;     // [rows] sticky `wide` byte: != 0 once any value of the row's state, or of a record it was handed, reached
                        // 2^30 -- such a row is evaluated by the 64-bit kernels only (raft_logic.cuh, narrow pass)
    u32*        q_used; // != 0 once any consistent-query state may be non-zero in this engine (see update_term_and_voted_for)
    u64*        lrs;    // [rows] start index of the LAST run (copy of run[n_runs-1].x; 0 when the log is
                        // empty): lets the step kernel load it together with the other pairs
    // transport / io.  Input record planes (mailboxes, locals) are TILED: plane p holds, for
    // every tile of 32 consecutive rows (one warp), 4 chunk sub-tiles [chunk j][lane] of
    // 16 bytes, i.e. the 2 KB a warp needs from a plane are contiguous (one cp.async.bulk) and
    // land in shared memory chunk-major (lane-consecutive 16-byte words: conflict-free LDS.128).
    ulonglong2* mbox[2];   // plane (src*DEPTH + k)
    u64*        mbox_cnt[2]; // [rows] one byte per sender slot
    ulonglong2* loc;       // plane k: host ("local") events
    u32*        loc_n;     // [rows]
    u32 tiles;             // ceil(rows / 32)
    ra_event* omsg;     // [k][rows] outgoing RPC records (non-routed)
    ra_note*  onote;    // [k][rows]
    u32*      out_n;    // [rows] msgs | notes << 16
    u64*      counters; // [RA_N_COUNTERS]: ra_counters' fields, the stall histogram, the reference's counters (raft_row.cuh)
    u32*      abort;    // != 0: a host batch was rejected (ra_engine_submit); the step kernels do nothing until the host has cleaned up
    u32 rows, groups, members;
    u32 groups_inv;        // floor(2^32 / groups)
    u32 max_pipeline, max_batch;
    u32 routed, pure;
    u32 note_cap;          // notes per row per step (<= RA_NOTE_CAP), see note_budget_ok()
    // cross-shard transport (n_shards > 1): member (g, s) lives on shard (g + s) mod N at local
    // group index g div N, so a record from slot s to slot t of the same group always goes to
    // shard (shard + t - s) mod N and to the SAME local row index t * groups + q there.
    u32 n_shards, shard;
    ra_event* outbox;      // [n_shards][out_cap] dense buckets, one per destination shard
    u32*      out_cnt;     // [n_shards]
    u32       out_cap;
    // peer transport: the mailbox buffers of every shard, mapped into this GPU's address space
    // (own shard included); records are stored straight into the destination GPU's HBM
    u32         peer_mode;
    ulonglong2* peer_mbox[2][8];
    u64*        peer_cnt[2][8];
};

#ifndef CTA_T
#define CTA_T 128                 // threads per CTA (4 independent warps)
#endif
#define RT 32                     // rows per record tile = one warp
// address (in 16-byte words) of chunk j of the record of `row` in tiled plane `plane`
__device__ __forceinline__ size_t rec_word(u32 tiles, u32 plane, u32 row, u32 j)
{
    return (((size_t)plane * tiles + (row >> 5)) * 4 + j) * RT + (row & (RT - 1));
}

struct FloodArgs { u32 on; u32 cmds; u32 permille; u32 drop; u32 withhold; u32 part; u32 part_len; u32 _p; u64 seed; u64 step; };

__device__ __forceinline__ ulonglong2 ld2(const ulonglong2* p) { return *p; }
__device__ __forceinline__ void st2(ulonglong2* p, u64 x, u64 y) { *p = make_ulonglong2(x, y); }

__device__ __forceinline__ u64 mix64(u64 x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}


// a stalled row's step context, handed from the step kernel to raft_general_kernel
struct StallCtx {                      // 4 x 16 bytes
    u32 row, flags, rem_mbox, rem_loc;
    u32 n_msgs_notes, status, sent_to, pn_type_slot_wk;
    u64 pn_a, pn_b;
    u64 pn_c;
    // Member::wk >> 16 -- the per-peer "sent a record that is not short" bits; pn_type_slot_wk keeps its low 16 bits.
    // A stalled row's end of step publishes them in the count bytes, which size the receiver's fetch in the next step,
    // so they must survive the stall.  The host emulation carries them the same way (tests/emu: step_row, general_row).
    union { u64 wk_hi; u64 _pad; };
};
#define STALL_PENDING 1u               // the deferred pipeline pass has not run yet
