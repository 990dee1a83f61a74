// Row-level pieces shared by the step kernels (engine.cu) and by the host-side emulation (tests/emu/): loading /
// writing back a row's registers and its end of step.  Included by raft_step.cuh inside each logic namespace.
__device__ __forceinline__ void member_init(Member& m, const Cols& C, u32 r, ulonglong2 tc, ulonglong2 lg, ulonglong2 lw,
                                            ulonglong2 ap, u64 lrs, int cur, ulonglong2* sp)
{
    m.C = &C; m.row = r;
    {   // slot = r / groups through the precomputed reciprocal floor(2^32 / groups): off by at most one
        u32 q = __umulhi(r, C.groups_inv), rem = r - q * C.groups;
        if (rem >= C.groups) { q++; rem -= C.groups; }
        if (rem >= C.groups) { q++; rem -= C.groups; }
        m.slot = q; m.group = rem;
    }
    // (plain truncation in the narrow pass: a row that does not fit is never evaluated there nor written back)
    m.term = (ix_t)tc.x; m.commit = (ix_t)tc.y; m.last_idx = (ix_t)lg.x; m.last_term = (ix_t)lg.y;
    m.lw_idx = (ix_t)lw.x; m.lw_term = (ix_t)lw.y; m.applied = (ix_t)ap.x; m.meta = ap.y;
    m.cold = 0;
    m.lrs = (ix_t)lrs; m.lrs_ok = MT_NRUNS(ap.y) ? 1u : 0u;
    m.n_msgs = 0; m.n_notes = 0; m.status = MT_ROLE(ap.y) << 16; m.wk = 0;
    m.sent_to = 0; m.pn_type = RA_NOTE_NONE; m.pn_slot = 0; m.pn_a = m.pn_b = m.pn_c = 0;
    m.c_pack = 0; m.c_ref = 0; m.c_commits = m.c_applied = 0;
    m.nb = cur ^ 1;
#ifdef RA_HOST_EMU
    m.sp = sp;
#else
    m.sp = (u32)__cvta_generic_to_shared(sp);
#endif
    m.pstate = 0; m.pipe_clean = 0;
}

// The four hot pairs change on practically every step of an active row (commit_index,
// last_index, last_written, last_applied / meta), so they are stored unconditionally: keeping
// their loaded values around just to skip a store costs 16 registers per thread.
__device__ __forceinline__ void member_writeback(const Member& m, const Cols& C, u32 r)
{
    st2(&C.tc[r], W(m.term), W(m.commit));
    st2(&C.lg[r], W(m.last_idx), W(m.last_term));
    st2(&C.lw[r], W(m.lw_idx), W(m.lw_term));
    st2(&C.ap[r], W(m.applied), m.meta);
    lrs_writeback(m);
#if RA_NARROW_PASS
    // the row's sticky `wide` byte: from 2^30 on its next steps belong to the 64-bit kernels
    if ((m.term | m.commit | m.last_idx | m.last_term | m.lw_idx | m.lw_term | m.applied) >= (ix_t)RA_NARROW_LIMIT) C.wf[r] = 1;
#endif
}

// ---- flood fault injection (include/ra_engine.h, ra_flood_faults): keyed by GLOBAL ids ---------------------
__device__ __forceinline__ void flood_ids(const Cols& C, const Member& m, u32 r, u64& gg, u64& gr)
{
    gg = m.group; gr = r;
    if (C.n_shards > 1) {
        gg = (u64)C.n_shards * m.group + (C.shard + 8u * C.n_shards - m.slot) % C.n_shards;
        gr = (u64)m.slot * C.groups * C.n_shards + gg;
    }
}
// is the mailbox record `e` lost before row r evaluates it in step F.step?
template <int MM>
__device__ __forceinline__ bool flood_lost(const FloodArgs& F, const Cols& C, const Member& m, u32 r, const Rec& e)
{
    if (!(F.drop | F.part)) return false;
    u64 gg, gr; flood_ids(C, m, r, gg, gr);
    const u32 from = R_from(e);
    if (F.part) {                                            // one member of the group is cut off in this window
        const u64 w = F.step / F.part_len;
        const u32 h = (u32)(mix64(F.seed ^ (w * 0xC2B2AE3D27D4EB4Full) ^ (gg * 0x165667B19E3779F9ull)) >> 32);
        if (h % 1000u < F.part) { const u32 p = (h / 1000u) % NMEM(C); if (p == m.slot || p == from) return true; }
    }
    if (F.drop && R_type(e) == RA_EV_AER) {
        const u32 h = (u32)(mix64(F.seed ^ (F.step * 0x9E3779B97F4A7C15ull) ^ (gr * 0xD6E8FEB86659FD93ull) ^ ((u64)(from + 1) << 56)) >> 32);
        if (h % 1000u < F.drop) return true;
    }
    return false;
}

// end of a row's step: publish mailbox counts, STATUS note, output counts, flood host model
// FAULTS = false compiles the fault injection out (the specialisations of the hot kernel that run the plain flood)
template <int MM, bool FAULTS = true>
__device__ __forceinline__ u32 row_end_of_step(Member& m, const Cols& C, u32 r, int cur, const FloodArgs& F)
{
    u32 fatal = 0;
    const bool routed = MTR == TR_RUNTIME ? (C.routed != 0) : (MTR != TR_HOST);
    if (routed) {
        const bool sharded = MTR == TR_RUNTIME ? (C.n_shards > 1) : (MTR == TR_PEER || MTR == TR_BUCKET);
        const bool peer = MTR == TR_RUNTIME ? (C.peer_mode != 0) : (MTR == TR_PEER);
        for (u32 s = 0; s < NMEM(C); s++) {
            if (s == m.slot) continue;
            u64* cnt = C.mbox_cnt[cur ^ 1];
            if (sharded) {
                const u32 ds = (C.shard + s + 8u * C.n_shards - m.slot) % C.n_shards;
                if (peer) cnt = C.peer_cnt[cur ^ 1][ds];                 // byte store over NVLink
                else if (ds != C.shard) continue;   // set when the records are delivered (deliver_kernel)
            }
            // (a count byte is zero when its buffer comes round again -- the owner clears the word when it consumes
            // it -- so only senders that sent something have to publish: 1 of a follower's 4 bytes in steady state)
            const u32 nsent = (m.sent_to >> (4 * s)) & 15u;
            if (nsent) reinterpret_cast<u8*>(&cnt[(size_t)s * C.groups + m.group])[m.slot] = (u8)(nsent | (((m.wk >> (16 + s)) & 1u) << 4));
        }
    }
    // record_leader_msg alone (the steady state of a follower) does not get a STATUS note of its own: the
    // flags ride in the aux field of the row's last note of the step (include/ra_engine.h, RA_NOTE_STATUS)
    const u32 st16 = m.status & 0xffffu;
    const bool elide = st16 == RA_ST_LEADER_MSG && m.pn_type != RA_NOTE_NONE;
    note_flush(m, elide ? st16 : 0u);
    if (st16 && !elide) {
        u64 ld = MT_LEADER(m.meta), vf = MT_VOTED(m.meta);
        u64 b = (vf == SLOT_NONE ? 0xFFull : vf) | ((ld == SLOT_NONE ? 0xFFull : ld) << 8) |
                ((u64)((m.status >> 16) & 7u) << 16) | ((u64)MT_ROLE(m.meta) << 24);
        note_store(m, m.n_notes, RA_NOTE_STATUS, m.slot, m.status & 0xffffu, W(m.term), b,
                   ((m.status >> 20) & 0xffu) | ((u64)(m.status >> 28) << 8));
        m.n_notes++;
        if (m.status & RA_ST_FATAL) fatal = 1;
    }
    C.out_n[r] = m.n_msgs | (m.n_notes << 16);
    // flood: synthetic host (DESIGN.md "flood host model")
    if (F.on && !MT_FATAL(m.meta)) {
        u32 k = 0, heads = 0;                               // heads: loc_n bits 12 + k, the records not written short
        bool held = false;                                  // a lagging fsync: this step's notifications are not produced
        if (FAULTS && F.withhold && (m.wk & 3u)) {
            u64 gg0, gr0; flood_ids(C, m, r, gg0, gr0);
            held = (u32)(mix64(F.seed ^ (F.step * 0xA0761D6478BD642Full) ^ (gr0 * 0xE7037ED1A0B428DBull)) >> 32) % 1000u < F.withhold;
        }
        if (held) m.wk = 0;
        // {written, Term, {From, To}} for the (last two) WAL_APPEND notes of this step: read back
        // from the row's own note slots instead of being carried in registers through the step
        if ((m.wk & 3u) == 2) {
            const ulonglong2* q = reinterpret_cast<const ulonglong2*>(&C.onote[(size_t)((m.wk >> 8) & 15u) * C.rows + r]);
            const ulonglong2 h = q[0], t = q[1];
            heads |= put_local(C.loc, C.tiles, k, r, RA_EV_WRITTEN, 0, 0, t.y, h.y, t.x) << (12 + k); k++;
        }
        if ((m.wk & 3u) >= 1) {
            const ulonglong2* q = reinterpret_cast<const ulonglong2*>(&C.onote[(size_t)((m.wk >> 4) & 15u) * C.rows + r]);
            const ulonglong2 h = q[0], t = q[1];
            heads |= put_local(C.loc, C.tiles, k, r, RA_EV_WRITTEN, 0, 0, t.y, h.y, t.x) << (12 + k); k++;
        }
        const u32 role = MT_ROLE(m.meta);
        if (role == RA_LEADER && F.cmds) { heads |= put_local(C.loc, C.tiles, k, r, RA_EV_COMMAND, 0, F.cmds, 0, 0, 0) << (12 + k); k++; }
        u32 idle = MT_IDLE(m.meta);
        if (role == RA_LEADER || (m.status & RA_ST_LEADER_MSG)) idle = 0;
        else if (idle < 15) idle++;
        bool fire = false;
        if (role != RA_LEADER) {
            // the model is keyed by GLOBAL group / row ids so that a sharded run equals the unsharded one
            u64 gg = m.group, gr = r;
            if (C.n_shards > 1) {
                gg = (u64)C.n_shards * m.group + (C.shard + 8u * C.n_shards - m.slot) % C.n_shards;
                gr = (u64)m.slot * C.groups * C.n_shards + gg;
            }
            if (F.permille) {
                const u32 h = (u32)(mix64(F.seed ^ (F.step * 0x9E3779B97F4A7C15ull) ^ (gg * 0xD1B54A32D192ED03ull)) >> 32);
                if ((h % 1000u) < F.permille && ((h / 1000u) % NMEM(C)) == m.slot) fire = true;
            }
            if (idle >= 8) {                                // the hash only matters from 8 idle steps on
                const u32 h2 = (u32)(mix64(F.seed ^ (gr * 0xA24BAED4963EE407ull) ^ F.step) >> 32);
                if (idle >= 8 + (h2 & 7u)) fire = true;
            }
        }
        if (fire) { heads |= put_local(C.loc, C.tiles, k, r, RA_EV_ELECTION_TIMEOUT, 0, 0, 0, 0, 0) << (12 + k); k++; idle = 0; }
        MT_SET(m.meta, 28, 4, idle);
        C.loc_n[r] = k | heads;
    }
    return fatal;
}

