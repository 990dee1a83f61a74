// What engine.cu and the host emulation (tests/emu/) share besides the step logic: conversions between a row of the
// column store and the ABI's ra_row_state, the bucket transport's delivery, the consistent-query rows and the ingest
// of a host batch (index-width independent: plain 64-bit copies), and the host-side rules of the C ABI: config,
// column layout, counter layout, argument checks, transport choice.
#pragma once
#include <stdlib.h>
#include <string.h>
#include "raft_step.cuh"

// ---- row <-> ra_row_state (load_rows / read_rows / reset_empty) -------------------------------
__device__ __forceinline__ void reset_row(const Cols& C, const u32 r)
{
    // ra_server_SUITE:empty_state/2: term 0, log {0 => 0}, peers next=1 match=0, all voters
    u64 meta = 0;
    MT_SET(meta, 0, 3, RA_FOLLOWER); MT_SET(meta, 3, 4, SLOT_NONE); MT_SET(meta, 7, 4, SLOT_NONE);
    MT_SET(meta, 19, 4, 1); MT_SET(meta, 27, 1, 1);
    MT_SET(meta, 56, 8, (1u << C.members) - 1u);
    st2(&C.tc[r], 0, 0); st2(&C.lg[r], 0, 0); st2(&C.lw[r], 0, 0); st2(&C.ap[r], 0, meta);
    st2(&C.sn[r], 0, 0); st2(&C.tk[r], 0, 0); st2(&C.fm[r], 0, 0);
    st2(&C.cd[r], 0, 0); st2(&C.cd[(size_t)C.rows + r], 0, 0);
    for (u32 s = 0; s < C.members; s++) { st2(&C.pnm[(size_t)s * C.rows + r], 1, 0); C.pcs[(size_t)s * C.rows + r] = 0; }
    for (u32 k = 0; k < RA_MAX_RUNS; k++) st2(&C.run[(size_t)k * C.rows + r], 0, 0);
    C.lrs[r] = 0;
    C.qi[r] = 0; C.qa[r] = 0; C.wc[r] = 0; C.wf[r] = 0;
    for (u32 s = 0; s < C.members; s++) C.pqi[(size_t)s * C.rows + r] = 0;
    C.loc_n[r] = 0; C.out_n[r] = 0;
    if (C.routed) { C.mbox_cnt[0][r] = 0; C.mbox_cnt[1][r] = 0; }
}

// does any index / term of a row state reach 2^30 (RA_NARROW_LIMIT)?  (device: load_row; host: ra_engine_load_rows
// counts them to choose the hot kernel)
__host__ __device__ __forceinline__ bool row_state_is_wide(const ra_row_state& s, u32 members)
{
    u64 big = s.current_term | s.commit_index | s.last_index | s.last_term | s.last_written_index | s.last_written_term |
              s.last_applied | s.snapshot_index | s.snapshot_term | s.pre_vote_token | s.token_counter | s.first_index |
              s.cond_reply_term | s.cond_reply_next_index | s.cond_reply_last_index | s.cond_reply_last_term;
    for (u32 p = 0; p < members && p < RA_MAX_MEMBERS; p++)
        big |= s.peers[p].next_index | s.peers[p].match_index | s.peers[p].commit_index_sent;
    for (u32 k = 0; k < s.n_runs && k < RA_MAX_RUNS; k++) big |= s.run_start[k] | s.run_term[k];
    return big >= 0x40000000ull;
}

__device__ __forceinline__ void load_row(const Cols& C, const ra_row_state& s)
{
    const u32 r = s.row;
    u64 meta = 0;
    MT_SET(meta, 0, 3, s.role);
    MT_SET(meta, 3, 4, s.leader_slot == RA_NO_SLOT ? SLOT_NONE : s.leader_slot);
    MT_SET(meta, 7, 4, s.voted_for == RA_NO_SLOT ? SLOT_NONE : s.voted_for);
    MT_SET(meta, 11, 2, s.membership); MT_SET(meta, 13, 2, s.condition);
    MT_SET(meta, 15, 4, s.votes); MT_SET(meta, 19, 4, s.n_runs);
    MT_SET(meta, 23, 1, s.has_snapshot ? 1 : 0);
    MT_SET(meta, 24, 1, (s.flags & 1) ? 1 : 0); MT_SET(meta, 25, 1, (s.flags & 2) ? 1 : 0);
    MT_SET(meta, 26, 1, (s.flags & 4) ? 1 : 0);
    MT_SET(meta, 27, 1, s.machine_version >= s.effective_machine_version ? 1 : 0);
    u32 voters = 0;
    for (u32 p = 0; p < RA_MAX_MEMBERS; p++) {
        MT_SET(meta, 32 + 3 * p, 3, s.peers[p].status);
        if (s.peers[p].voter) voters |= 1u << p;
    }
    MT_SET(meta, 56, 8, voters);
    st2(&C.tc[r], s.current_term, s.commit_index);
    st2(&C.lg[r], s.last_index, s.last_term);
    st2(&C.lw[r], s.last_written_index, s.last_written_term);
    st2(&C.ap[r], s.last_applied, meta);
    st2(&C.sn[r], s.snapshot_index, s.snapshot_term);
    st2(&C.tk[r], s.pre_vote_token, s.token_counter);
    st2(&C.fm[r], s.first_index, (u64)s.machine_version | ((u64)s.effective_machine_version << 32));
    st2(&C.cd[r], s.cond_reply_term, s.cond_reply_next_index);
    st2(&C.cd[(size_t)C.rows + r], s.cond_reply_last_index, s.cond_reply_last_term);
    for (u32 p = 0; p < C.members; p++) {
        st2(&C.pnm[(size_t)p * C.rows + r], s.peers[p].next_index, s.peers[p].match_index);
        C.pcs[(size_t)p * C.rows + r] = s.peers[p].commit_index_sent;
    }
    for (u32 k = 0; k < RA_MAX_RUNS; k++)
        st2(&C.run[(size_t)k * C.rows + r], k < s.n_runs ? s.run_start[k] : 0, k < s.n_runs ? s.run_term[k] : 0);
    C.lrs[r] = s.n_runs ? s.run_start[s.n_runs - 1] : 0;
    // the sticky `wide` byte (raft_logic.cuh, narrow pass): does every index / term of the row fit below 2^30?
    C.wf[r] = row_state_is_wide(s, C.members) ? 1 : 0;
    C.qi[r] = 0; C.qa[r] = 0; C.wc[r] = 0;
    for (u32 p = 0; p < C.members; p++) C.pqi[(size_t)p * C.rows + r] = 0;
    C.loc_n[r] = 0;
    // a (re)loaded member starts with an empty mailbox: records still in flight to it (both buffers, every sender)
    // were addressed to its earlier life.  (A fatal row never consumes its counts, so they can be many steps old.)
    if (C.routed) { C.mbox_cnt[0][r] = 0; C.mbox_cnt[1][r] = 0; }
}

__device__ __forceinline__ void read_row(const Cols& C, ra_row_state& s)
{
    const u32 r = s.row;
    const ulonglong2 tc = C.tc[r], lg = C.lg[r], lw = C.lw[r], ap = C.ap[r], sn = C.sn[r], tk = C.tk[r], fm = C.fm[r];
    const u64 meta = ap.y;
    s.role = MT_ROLE(meta); s.self_slot = r / C.groups; s.n_members = C.members;
    u32 l = MT_LEADER(meta), v = MT_VOTED(meta);
    s.leader_slot = l == SLOT_NONE ? RA_NO_SLOT : l; s.voted_for = v == SLOT_NONE ? RA_NO_SLOT : v;
    s.membership = MT_MEMBERSHIP(meta); s.condition = MT_COND(meta); s.has_snapshot = MT_HAS_SNAP(meta);
    s.votes = MT_VOTES(meta); s.machine_version = (u32)fm.y; s.effective_machine_version = (u32)(fm.y >> 32);
    s.n_runs = MT_NRUNS(meta);
    s.flags = MT_PIPE_PEND(meta) | (MT_COND_VALID(meta) << 1) | (MT_FATAL(meta) << 2);
    s.current_term = tc.x; s.commit_index = tc.y; s.last_applied = ap.x;
    s.pre_vote_token = tk.x; s.token_counter = tk.y;
    s.first_index = fm.x; s.last_index = lg.x; s.last_term = lg.y;
    s.last_written_index = lw.x; s.last_written_term = lw.y;
    s.snapshot_index = sn.x; s.snapshot_term = sn.y;
    for (u32 k = 0; k < RA_MAX_RUNS; k++) {
        ulonglong2 rr = C.run[(size_t)k * C.rows + r];
        s.run_start[k] = k < s.n_runs ? rr.x : 0; s.run_term[k] = k < s.n_runs ? rr.y : 0;
    }
    ulonglong2 c0 = C.cd[r], c1 = C.cd[(size_t)C.rows + r];
    s.cond_reply_term = c0.x; s.cond_reply_next_index = c0.y; s.cond_reply_last_index = c1.x; s.cond_reply_last_term = c1.y;
    for (u32 p = 0; p < RA_MAX_MEMBERS; p++) {
        ra_peer_init& pi = s.peers[p];
        if (p < C.members) {
            ulonglong2 nm = C.pnm[(size_t)p * C.rows + r];
            pi.next_index = nm.x; pi.match_index = nm.y; pi.commit_index_sent = C.pcs[(size_t)p * C.rows + r];
            pi.status = MT_PSTATUS(meta, p); pi.voter = MT_VOTER(meta, p);
        } else { pi.next_index = pi.match_index = pi.commit_index_sent = 0; pi.status = 0; pi.voter = 0; }
        for (int q = 0; q < 6; q++) pi._pad[q] = 0;
    }
}

// raft_general_kernel, after a row's step: the row turns `wide` (for good) once a record it was handed or one of its
// registers reaches 2^30.  Everything the general path writes into a row's state comes from those two sources (or
// from counters that grow by one per election), so a row whose byte is clear holds no larger value anywhere.
// (A pre_vote's d field is version | machine_version << 32: compared, never stored -- left out.)
__device__ __forceinline__ u64 rec_magnitude(const Rec& e)
{ return R_term(e) | R_a(e) | R_b(e) | R_c(e) | R_e(e) | (R_type(e) == RA_EV_PRE_VOTE ? 0ull : R_d(e)); }
__device__ __forceinline__ void row_mark_wide(const Cols& C, u32 r, const Member& m, u64 big)
{
    big |= m.term | m.commit | m.last_idx | m.last_term | m.lw_idx | m.lw_term | m.applied;
    if (big >= RA_NARROW_LIMIT) C.wf[r] = 1;
}

// ---- bucket transport: one record another shard sent to a member of this engine ---------------
// -> mailbox plane of the next step.  The slot is fixed by the record itself (sender slot, k-th
// record of that sender for this row); byte `from` of the row's count word becomes
// max(old count, k + 1) | tail flag (bit 3) | not-short flag (bit 4).
__device__ __forceinline__ void deliver_record(const Cols& C, const int buf, const Rec& r)
{
    const u32 row = R_row(r), from = R_from(r), k = (u32)(r.w0.y >> 32);
    if (row >= C.rows || from >= C.members || k >= RA_MBOX_DEPTH) return;
    const u32 f = st_rec_plane(C.mbox[buf], C.tiles, from * RA_MBOX_DEPTH + k, row, r);
    const u32 size = ((f & RF_TAIL) << 2) | ((f & RF_NOT_SHORT) << 4);
    u32* w = reinterpret_cast<u32*>(&C.mbox_cnt[buf][row]) + (from >> 2);
    const u32 sh = 8u * (from & 3u);
    u32 old = *w;
    for (;;) {
        const u32 ob = (old >> sh) & 0xffu;
        const u32 nb = ((ob & 7u) >= k + 1 ? (ob & 7u) : k + 1) | (ob & 0x18u) | size;
        if (nb == ob) break;
        const u32 seen = atomicCAS(w, old, (old & ~(0xffu << sh)) | (nb << sh));
        if (seen == old) break;
        old = seen;
    }
}

// ---- ingest: a flat host batch -> the per-row local slots --------------------------------------
// The two record forms of a host batch: which types each may carry, and how one record is stored as the k-th local
// record of its row, returning its loc_n size bits for k = 0 (8 + k: tail, 12 + k: not short).
// 64-byte ra_event: any event type, stored as it is, from a slot below 15 or RA_NO_SLOT (a row keeps leader_id and
// voted_for in 4 bits: slot 17 would be read as slot 1, include/ra_engine.h at ra_event.from_slot).
__device__ __forceinline__ bool ingest_type_ok(const ra_event& ev)
{
    return ev.type <= RA_EV_CONSISTENT_QUERY && ev.type != RA_EV_NONE && (ev.from_slot < 15u || ev.from_slot == RA_NO_SLOT);
}
__device__ __forceinline__ u32 ingest_store(const Cols& C, u32 k, u32 row, const ra_event& ev)
{
    const u32 f = st_rec_plane(C.loc, C.tiles, k, row, ld_rec(&ev));
    return ((f & RF_TAIL) << 7) | ((f & RF_NOT_SHORT) << 12);
}
// 32-byte ra_host_event: host-origin types only (no RPC), every record RS_PLAIN
__device__ __forceinline__ bool ingest_type_ok(const ra_host_event& ev)
{
    const u32 t = ev.type;
    return t == RA_EV_WRITTEN || t == RA_EV_COMMAND || t == RA_EV_ELECTION_TIMEOUT || t == RA_EV_AWAIT_COND_TIMEOUT ||
           t == RA_EV_PIPELINE_RPCS || t == RA_EV_TICK || t == RA_EV_CONSISTENT_QUERY;
}
__device__ __forceinline__ u32 ingest_store(const Cols& C, u32 k, u32 row, const ra_host_event& ev)
{
    const ulonglong2* src = reinterpret_cast<const ulonglong2*>(&ev);
    const ulonglong2 h = src[0], t = src[1];                   // {row | type<<32 | flags<<40 | n<<48, term}, {a, b}
    const u32 type = (u32)(h.x >> 32) & 0xffu, flags = (u32)(h.x >> 40) & 0xffu, nn = (u32)(h.x >> 48);
    return put_local(C.loc, C.tiles, k, row, type, flags, nn, h.y, t.x, t.y) << 12;
}

#ifdef RA_HOST_EMU
// the host emulation (tests/emu) runs ingest_event one event at a time: plain read-modify-writes
static inline u32 atomicMax(u32* p, u32 v) { const u32 o = *p; if (v > o) *p = v; return o; }
static inline u32 atomicOr(u32* p, u32 v) { const u32 o = *p; *p = o | v; return o; }
#endif
// Event i of a batch of n: the head of a row's run stores the run into the row's local slots.  *err becomes at least
// 1 = ungrouped, 2 = too many for a row, 3 = bad row or type.  ingest_kernel runs it once per thread, the host
// emulation for i = 0 .. n - 1 in turn: each row has one run head and the errors combine with max, so the order
// does not change the result.
template <typename EV>
__device__ __forceinline__ void ingest_event(const Cols& C, const EV* ev, u32 n, u32 i, u32* err)
{
    const u32 row = ev[i].row;
    if (row >= C.rows || !ingest_type_ok(ev[i])) { atomicMax(err, 3u); return; }
    if (i > 0 && ev[i - 1].row == row) return;                 // not the head of its run
    u32 len = 1;
    while (i + len < n && ev[i + len].row == row && len <= RA_LOCAL_CAP) len++;
    if (len > RA_LOCAL_CAP) { atomicMax(err, 2u); return; }
    if (atomicCAS(&C.loc_n[row], 0u, len) != 0u) { atomicMax(err, 1u); return; }
    u32 size = 0;
    for (u32 k = 0; k < len; k++) size |= ingest_store(C, k, row, ev[i + k]) << k;
    if (size) atomicOr(&C.loc_n[row], size);
}

// ---- consistent-query state of a row <-> ra_query_state ----------------------------------------
__device__ __forceinline__ void load_query_row(const Cols& C, const ra_query_state& q)
{
    const u32 r = q.row;
    *C.q_used = 1u;
    C.qi[r] = q.query_index; C.qa[r] = q.agreed_index;
    for (u32 p = 0; p < C.members; p++) C.pqi[(size_t)p * C.rows + r] = q.peer_query_index[p];
}
__device__ __forceinline__ void read_query_row(const Cols& C, ra_query_state& q)
{
    const u32 r = q.row;
    q._pad = 0; q.query_index = C.qi[r]; q.agreed_index = C.qa[r];
    for (u32 p = 0; p < RA_MAX_MEMBERS; p++) q.peer_query_index[p] = p < C.members ? C.pqi[(size_t)p * C.rows + r] : 0;
}

// ---- Cols::counters ----------------------------------------------------------------------------
// [0, RA_CNT_STALL) ra_counters' aggregate fields, events .. fatal_rows;  [RA_CNT_STALL, RA_CNT_REF) the stall
// histogram, role x type: events that left the hot kernel;  [RA_CNT_REF, RA_N_COUNTERS) the reference's per-path
// counters in the order of Member::c_ref (CR_*)
#define RA_CNT_STALL 8
#define RA_CNT_REF (RA_CNT_STALL + 8 * 16)
#define RA_N_COUNTERS (RA_CNT_REF + 8)
__device__ __forceinline__ u32 cnt_stall(u32 role, u32 type) { return RA_CNT_STALL + (role & 7u) * 16 + (type & 15u); }

static inline void counters_unpack(const u64* h, u64 steps, ra_counters* out)
{
    out->events = h[0]; out->commits = h[1]; out->applied = h[2]; out->msgs_out = h[3];
    out->msgs_dropped = h[4]; out->elections_won = h[5]; out->fatal_rows = h[6]; out->steps = steps;
    out->aer_received_follower = h[RA_CNT_REF + 0]; out->aer_received_follower_empty = h[RA_CNT_REF + 1];
    out->aer_replies_success = h[RA_CNT_REF + 2]; out->aer_replies_failed = h[RA_CNT_REF + 3];
    out->elections = h[RA_CNT_REF + 4]; out->pre_vote_elections = h[RA_CNT_REF + 5];
    out->term_and_voted_for_updates = h[RA_CNT_REF + 6];
}

// ---- ra_engine_create ----------------------------------------------------------------------------
// RA_E_INVAL for a config no engine accepts, else `out` = the config with its defaults and narrow_mode = the hot
// kernel RA_STEP_WIDE asks for: unset = 0 (auto), "0" = 1 (always the 32-bit one), else 2 (never)
static inline int cfg_resolve(const ra_engine_cfg* cfg, ra_engine_cfg& out, int& narrow_mode)
{
    if (!cfg || cfg->n_members < 1 || cfg->n_members > RA_MAX_MEMBERS || cfg->n_groups == 0) return RA_E_INVAL;
    if ((u64)cfg->n_groups * cfg->n_members > 0x7fffffffull) return RA_E_INVAL;
    if (cfg->n_shards > 1 && (!cfg->route_on_device || cfg->shard >= cfg->n_shards || cfg->n_shards > 64)) return RA_E_INVAL;
    if (cfg->note_cap && (cfg->note_cap < RA_NOTE_RESERVE + 2 || cfg->note_cap > RA_NOTE_CAP)) return RA_E_INVAL;
    out = *cfg;
    if (out.max_pipeline_count == 0) out.max_pipeline_count = 4096;
    if (out.max_aer_batch == 0) out.max_aer_batch = 128;
    const char* w = getenv("RA_STEP_WIDE");
    narrow_mode = !(w && *w) ? 0 : (*w == '0' ? 1 : 2);
    return RA_OK;
}

#define RA_BAR_WORDS 64                       // barrier flag words behind mbox_cnt[b] (one per source shard)
// The column store of an engine with config `cfg` (defaults filled in): the scalar fields, and every column at its
// size through the caller's allocator, alloc(T*& p, size_t count) -> RA_OK, which also zeroes it.  Everything else
// (the transports' buffers, Cols::abort) starts null.
template <typename Alloc>
static inline int cols_init(Cols& C, const ra_engine_cfg& cfg, Alloc alloc)
{
    const size_t R = (size_t)cfg.n_groups * cfg.n_members, M = cfg.n_members;
    C = Cols{};
    C.rows = (u32)R; C.groups = cfg.n_groups; C.members = cfg.n_members;
    C.groups_inv = cfg.n_groups > 1 ? (u32)(0x100000000ull / cfg.n_groups) : 0xFFFFFFFFu;
    C.max_pipeline = cfg.max_pipeline_count; C.max_batch = cfg.max_aer_batch;
    C.routed = cfg.route_on_device ? 1 : 0; C.pure = cfg.pure ? 1 : 0;
    C.note_cap = cfg.note_cap ? cfg.note_cap : RA_NOTE_CAP;
    C.n_shards = cfg.n_shards > 1 ? cfg.n_shards : 1; C.shard = cfg.n_shards > 1 ? cfg.shard : 0;
    C.tiles = (u32)((R + RT - 1) / RT);
    const size_t PW = (size_t)C.tiles * 4 * RT;             // 16-byte words per tiled plane
    int rc;
#define CA(p, n) if ((rc = alloc(p, (n))) != RA_OK) return rc
    CA(C.tc, R); CA(C.lg, R); CA(C.lw, R); CA(C.ap, R); CA(C.sn, R); CA(C.tk, R); CA(C.fm, R);
    CA(C.cd, 2 * R); CA(C.pnm, M * R); CA(C.pcs, M * R); CA(C.run, RA_MAX_RUNS * R); CA(C.lrs, R);
    CA(C.qi, R); CA(C.qa, R); CA(C.pqi, M * R); CA(C.q_used, 4); CA(C.wc, R); CA(C.wf, R);
    CA(C.loc, (size_t)RA_LOCAL_CAP * PW); CA(C.loc_n, R);
    CA(C.onote, (size_t)RA_NOTE_CAP * R); CA(C.out_n, R + 1); CA(C.counters, RA_N_COUNTERS);   // out_n[R] stays 0: the scan's total
    CA(C.omsg, (size_t)RA_MSG_CAP * (C.routed && !C.pure ? 1 : R));   // routed records stay on the device
    // + RA_BAR_WORDS: the peer transport's step barrier flags live behind the counts of buffer 0,
    // so they are covered by the IPC mapping the peers already have
    for (int b = 0; b < 2 && C.routed; b++) { CA(C.mbox[b], M * RA_MBOX_DEPTH * PW); CA(C.mbox_cnt[b], R + RA_BAR_WORDS); }
#undef CA
    return RA_OK;
}

// ---- argument checks of the row calls ------------------------------------------------------------
// an array of per-row structs (ra_row_state, ra_query_state) unless n = 0, every one for a row of this engine
template <typename T>
static inline bool rows_ok(const Cols& C, const T* rows, size_t n)
{
    if (!rows && n) return false;
    for (size_t i = 0; i < n; i++) if (rows[i].row >= C.rows) return false;
    return true;
}
// ra_engine_load_rows: every state valid for this engine.  A bulk load (at least half the rows) in auto mode
// (narrow_mode 0) chooses the hot kernel: the 32-bit one unless most of the states reach 2^30.
static inline int load_rows_check(const Cols& C, const ra_row_state* rows, size_t n, int narrow_mode, int& narrow)
{
    if (!rows_ok(C, rows, n)) return RA_E_INVAL;
    for (size_t i = 0; i < n; i++)
        if (rows[i].n_members != C.members || !ra_row_state_valid(&rows[i])) return RA_E_INVAL;
    if (narrow_mode == 0 && n * 2 >= C.rows) {
        size_t wide = 0;
        for (size_t i = 0; i < n; i++) wide += row_state_is_wide(rows[i], C.members) ? 1 : 0;
        narrow = wide * 2 < n;
    }
    return RA_OK;
}

// ra_engine_submit_host_segs: at most RA_MAX_SEGS pieces, each an array unless it is empty
#define RA_MAX_SEGS 256
static inline bool host_segs_ok(const ra_host_event_seg* segs, size_t n_segs)
{
    if (n_segs > RA_MAX_SEGS || (!segs && n_segs)) return false;
    for (size_t k = 0; k < n_segs; k++) if (!segs[k].ev && segs[k].n) return false;
    return true;
}

// ---- transports ------------------------------------------------------------------------------------
// where a step's RPC records go (MK_MM): the step kernels are specialised by it
static inline int step_transport(const Cols& C)
{
    return !C.routed ? TR_HOST : (C.n_shards > 1 ? (C.peer_mode ? TR_PEER : TR_BUCKET) : TR_LOCAL);
}

// ra_engine_flood_faults: the step kernels' FloodArgs for its arguments (F.step is set per step); the flood runs on
// routed engines only, and a partition needs a length
static inline int flood_args(const Cols& C, const ra_flood_faults* ff, u32 cmds, u32 permille, u64 seed, FloodArgs& F)
{
    if (!C.routed || (ff && ff->partition_permille && !ff->partition_steps)) return RA_E_INVAL;
    memset(&F, 0, sizeof F);
    F.on = 1; F.cmds = cmds; F.permille = permille; F.seed = seed;
    if (ff) { F.drop = ff->drop_permille; F.withhold = ff->withhold_permille; F.part = ff->partition_permille; F.part_len = ff->partition_steps; }
    return RA_OK;
}

// the bucket transport (ra_engine_set_outbox, ra_engine_deliver)
static inline int cols_set_outbox(Cols& C, void* outbox, uint32_t* counts, uint32_t cap)
{
    if (C.n_shards < 2 || !outbox || !counts || !cap) return RA_E_INVAL;
    C.outbox = (ra_event*)outbox; C.out_cnt = counts; C.out_cap = cap;
    return RA_OK;
}
static inline bool deliver_args_ok(const Cols& C, const void* inbox, const uint32_t* counts, uint32_t cap)
{
    return C.n_shards >= 2 && inbox && counts && cap;
}

// the peer transport (ra_engine_peer_get, ra_engine_peer_set): peer mode once every shard's buffers are known
static inline int cols_peer_get(const Cols& C, ra_peer_ptrs* out)
{
    if (!out || !C.routed) return RA_E_INVAL;
    for (int b = 0; b < 2; b++) { out->mbox[b] = C.mbox[b]; out->mbox_cnt[b] = C.mbox_cnt[b]; }
    return RA_OK;
}
static inline int cols_peer_set(Cols& C, uint32_t shard, const ra_peer_ptrs* p)
{
    if (!p || C.n_shards < 2 || C.n_shards > 8 || shard >= C.n_shards) return RA_E_INVAL;
    for (int b = 0; b < 2; b++) { C.peer_mbox[b][shard] = (ulonglong2*)p->mbox[b]; C.peer_cnt[b][shard] = (u64*)p->mbox_cnt[b]; }
    for (int b = 0; b < 2; b++) { C.peer_mbox[b][C.shard] = C.mbox[b]; C.peer_cnt[b][C.shard] = C.mbox_cnt[b]; }
    bool all = true;
    for (u32 k = 0; k < C.n_shards; k++) all = all && C.peer_mbox[0][k] && C.peer_mbox[1][k] && C.peer_cnt[0][k] && C.peer_cnt[1][k];
    C.peer_mode = all ? 1 : 0;
    return RA_OK;
}
