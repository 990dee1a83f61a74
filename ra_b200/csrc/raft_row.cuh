// Conversions between a row of the column store and the ABI's ra_row_state, the bucket transport's delivery and the
// consistent-query rows: index-width independent (plain 64-bit copies), shared by engine.cu and tests/emu/.
#pragma once
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
