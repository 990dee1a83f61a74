// raft_step_kernel -- the hot kernel of a step (see engine.cu for the frame it lives in: StepSmem, the TMA / mbarrier
// helpers, the counter flushes).  Included by engine.cu inside namespace ra_wide and inside namespace ra_narrow.
#if RA_NARROW_PASS
#define RA_STEP_MINB MINB_NARROW
#else
#define RA_STEP_MINB MINB
#endif
template <int MM, bool FAULTS>
__global__ void __launch_bounds__(CTA_T, RA_STEP_MINB)
raft_step_kernel(const __grid_constant__ Cols C, const int cur, const FloodArgs F,
                 StallCtx* __restrict__ stall_list, u32* __restrict__ stall_count, u32* __restrict__ stall_count_next)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    typedef StepSmem<MM, RA_NARROW_PASS != 0> Smem;
    Smem& S = *reinterpret_cast<Smem*>(smem_raw);
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    TL(__shared__ u64 tl_acc[WARPS][TL_WORDS]; const u64 tl_g0 = tl_gtime(), tl_c0 = clock64();)
    const u32 wtile = blockIdx.x * WARPS + warp;                 // this warp's record tile
    const u32 r = wtile * RT + lane;
    const bool valid = r < C.rows;
    u32 k_events = 0, k_commits = 0, k_applied = 0, k_msgs = 0, k_dropped = 0, k_elect = 0, k_fatal = 0;
    u64 k_ref = 0;
    grid_dep_wait();                                            // nothing of the previous kernel is read before this
    if (blockIdx.x == 0 && tid == 0) *stall_count_next = 0;    // the list of the step after this one

    // ---- what does this row have to do? ---------------------------------------------------
    // every per-row input of the step is requested up front, in one round trip to HBM
    const ulonglong2 z2 = make_ulonglong2(0, 0);
    ulonglong2 ap = z2, tc = z2, lg = z2, lw = z2;
    u64 cntw = 0, lrs = 0; u32 nloc = 0;
#if RA_NARROW_PASS
    u32 wfb = 0;                                                // the row's sticky `wide` byte (Cols::wf)
#endif
    if (valid) {
        ap = C.ap[r];
        nloc = C.loc_n[r];
#if RA_NARROW_PASS
        wfb = C.wf[r];
#endif
        if (C.routed) cntw = C.mbox_cnt[cur][r];
        tc = C.tc[r]; lg = C.lg[r]; lw = C.lw[r]; lrs = C.lrs[r];
    }
    if (*C.abort) return;                                       // a host batch was rejected: nothing may change
    const bool fatal0 = MT_FATAL(ap.y) != 0;
    const bool pending = valid && MT_PIPE_PEND(ap.y) != 0;
    // planes of this row: mailbox plane (sender s, depth k) = bit s * DEPTH + k, host slot k = bit NPM + k
    constexpr u32 NPM = (MMEM ? MMEM : RA_MAX_MEMBERS) * RA_MBOX_DEPTH;
    typedef typename PlaneMask<(NPM + RA_LOCAL_CAP <= 32)>::type mask_t;
    mask_t mine = 0;
    // senders (bits 0..7) / host slots (8..11) whose records carry a 32-byte tail, and the same + 16: whose
    // records are not all short
    u32 my_tail = 0;
    if (valid && !fatal0) {
        u32 mb = 0;
        for (u32 s = 0; s < NMEM(C); s++) {
            const u32 c = (u32)(cntw >> (8 * s)) & 0xffu;
            mb |= ((1u << (c & 7u)) - 1u) << (RA_MBOX_DEPTH * s);
            my_tail |= (((c >> 3) & 1u) | (((c >> 4) & 1u) << 16)) << s;
        }
        mine = (mask_t)mb | ((mask_t)((1u << (nloc & 7u)) - 1u) << NPM);
        my_tail |= (nloc & 0x0f00u) | ((nloc & 0xf000u) << 12);
    }
    const bool work = valid && (F.on || nloc || cntw || pending);
    // everything below is per warp: no CTA-wide barrier anywhere in this kernel
    mask_t todo = mask_or_warp(mine);                           // planes still to consume
    const u32 w_tail = __reduce_or_sync(0xffffffffu, my_tail);
    if (!__any_sync(0xffffffffu, work)) return;                 // whole warp idle
    TL(const u64 tl_g1 = tl_gtime(), tl_c1 = clock64();
       tl_acc[warp][lane] = 0; tl_acc[warp][lane + 32] = 0; __syncwarp();
       const u32 tl_lead = __popc(__ballot_sync(0xffffffffu, valid && MT_ROLE(ap.y) == RA_LEADER));)
    u64* bars = &S.bars[warp][0];
    if (lane == 0) {
        for (int i = 0; i < NST; i++) mbar_init(&bars[i], 1);
        mbar_fence_init();
    }
    __syncwarp();

    Member m;
#if RA_NARROW_PASS
    member_init(m, C, valid ? r : 0, tc, lg, lw, ap, lrs, cur, reinterpret_cast<ulonglong2*>(reinterpret_cast<uint2*>(S.peers_nm) + tid));
#else
    member_init(m, C, valid ? r : 0, tc, lg, lw, ap, lrs, cur, &S.peers_nm[tid]);
#endif
    m.row = r;
#if RA_NARROW_PASS
    const bool wide_row = wfb != 0;     // some value of this row does not fit 32-bit arithmetic: the general kernel's
#else
    const bool wide_row = false;
#endif
    if (work && !fatal0 && !wide_row && MT_ROLE(ap.y) == RA_LEADER) peers_prefetch<MM>(m);

    bool stalled = false;
    u32 stall_flags = 0;

    // ---- inputs: TMA stages this warp's record tiles (512 B, 1 KB or 2 KB of each) through a ring of NST 2 KB slots, in
    // evaluation order: deferred pipeline pass, mailbox planes by sender slot then depth, then
    // the host-event planes.  A slot is refilled as soon as the warp has consumed it.
    mask_t rem = 0;                                             // a stalled row's planes not yet evaluated
    if (work && ((!fatal0 && pending) || wide_row)) {           // pipeline_rpcs is not a fast path
        stalled = true; stall_flags = (!fatal0 && pending) ? STALL_PENDING : 0u; rem = mine;
    }
    mask_t toissue = todo;                                      // planes still to request
    u32 n_issued = 0, n_done = 0, st_issue = 0, st = 0, par = 0; // ring positions = counters mod NST, phase parity
#pragma unroll 1
    while (todo) {
        TL(const u64 tl_a = clock64();)
        if (lane == 0) {
#pragma unroll 1
            while (toissue && n_issued < n_done + NST) {
                const u32 q = mask_ffs(toissue); toissue &= toissue - 1;
                // (the tile address is rebuilt per issue -- a handful of integer ops in one lane -- instead of
                // holding two 64-bit plane bases in registers through the whole event loop)
                const size_t plane_words = (size_t)C.tiles * (4 * RT);      // 16-byte words per plane
                const ulonglong2* src = (q < NPM ? C.mbox[cur] + (size_t)q * plane_words
                                                 : C.loc + (size_t)(q - NPM) * plane_words) + (size_t)wtile * (4 * RT);
                const u32 tbit = q < NPM ? q / RA_MBOX_DEPTH : 8u + q - NPM;
                // chunk 0 (512 B) for short records only, 0 + 1 for heads, all four for tails (a tail is not short)
                const u32 bytes = (TILE_BYTES / 4) << (((w_tail >> tbit) & 1u) + ((w_tail >> (tbit + 16)) & 1u));
                fence_proxy_async();                            // the slot was read through the generic proxy
                mbar_expect_tx(&bars[st_issue], bytes);
                tma_load_tile(&S.stage[warp][st_issue][0], src, bytes, &bars[st_issue]);
                n_issued++; st_issue = st_issue + 1 == NST ? 0 : st_issue + 1;
            }
        }
        TL(const u64 tl_b = clock64();)
        const u32 p = mask_ffs(todo); todo &= todo - 1;
        const bool my = !stalled && ((mine >> p) & 1u);
        mbar_wait(&bars[st], par);
        TL(const u64 tl_c = clock64(); u64 tl_d = tl_c; u32 tl_t = 15;)
        if (my) {
            const ulonglong2* sp = &S.stage[warp][st][0];
            const ulonglong2 c0 = sp[lane], c1 = sp[RT + lane];
            ulonglong2 t2 = make_ulonglong2(0, 0), t3 = t2;
            if (rec_has_tail(c0)) { t2 = sp[2 * RT + lane]; t3 = sp[3 * RT + lane]; }
            Rec e;
            const bool fits = rec_decode(c0, c1, t2, t3, r, e);  // (narrow pass: every field below 2^30)
            TL(tl_d = clock64(); tl_t = R_type(e) & 15u;)
            if (MT_FATAL(m.meta)) m.c_pack += 1u;
            else if (FAULTS && p < NPM && flood_lost<MM>(F, C, m, r, e)) m.c_pack += 1u << 20;   // fault injection: lost in transit
            else if (!fits || !note_budget_ok(m) || C.pure || !fast_event<MM>(m, e)) {
                stalled = true;                                 // planes are consumed in bit order:
                rem = mine & ~(((mask_t)1 << p) - 1);           // p and up are left for the general kernel
                atomicAdd(&C.counters[cnt_stall(m_role(m), R_type(e))], 1ull);   // diagnostics
            }
        }
        TL(if (lane == 0) {
               u64* a = tl_acc[warp]; const u64 tl_e = clock64();
               a[10] += tl_b - tl_a; a[11] += tl_c - tl_b; a[12] += tl_d - tl_c; a[13]++;
               a[18 + 2 * tl_t] += tl_e - tl_d; a[19 + 2 * tl_t]++;
           })
        n_done++;
        if (++st == NST) { st = 0; par ^= 1u; }
        __syncwarp();                                           // every lane is done with the slot
    }
    TL(const u64 tl_g2 = tl_gtime(), tl_c2 = clock64(); u64 tl_t0 = 0, tl_t1 = 0, tl_t2 = 0, tl_t3 = 0;)
    const u32 rem_mbox = (u32)(rem & (((mask_t)1 << (NPM - 1) << 1) - 1)), rem_loc = (u32)(rem >> (NPM - 1) >> 1);

    if (work) {
        if (cntw && !fatal0) C.mbox_cnt[cur][r] = 0;
        if (nloc) C.loc_n[r] = 0;
        if ((m.pstate & 3u) == 2u) asm volatile("cp.async.wait_all;" ::: "memory");   // prefetch never consumed
        TL(tl_t0 = clock64();)
        peers_writeback<MM>(m);
        TL(tl_t1 = clock64();)
        if (!stalled) k_fatal = row_end_of_step<MM, FAULTS>(m, C, r, cur, F);
        TL(tl_t2 = clock64();)
        if (!wide_row) member_writeback(m, C, r);               // (a wide row's registers were never valid here)
        TL(tl_t3 = clock64();)
        k_events = m.c_pack & 0xffu; k_commits = m.c_commits; k_applied = m.c_applied;
        k_msgs = (m.c_pack >> 8) & 0xffu; k_dropped = m.c_pack >> 20; k_elect = (m.c_pack >> 16) & 15u;
        k_ref = m.c_ref;
    }
    // stalled rows: hand the rest of the step to raft_general_kernel
    const u32 sm = __ballot_sync(0xffffffffu, stalled);
    if (sm) {
        u32 base = 0;
        if (lane == 0) base = atomicAdd(stall_count, (u32)__popc(sm));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (stalled) {
            ulonglong2* q = reinterpret_cast<ulonglong2*>(&stall_list[base + __popc(sm & ((1u << lane) - 1u))]);
            q[0] = make_ulonglong2((u64)r | ((u64)stall_flags << 32), (u64)rem_mbox | ((u64)rem_loc << 32));
            q[1] = make_ulonglong2((u64)(m.n_msgs | (m.n_notes << 16)) | ((u64)m.status << 32),
                                   (u64)m.sent_to | ((u64)(m.pn_type | (m.pn_slot << 8) | (m.wk << 16)) << 32));
            q[2] = make_ulonglong2(W(m.pn_a), W(m.pn_b));
            q[3] = make_ulonglong2(W(m.pn_c), (u64)(m.wk >> 16));
        }
    }
    flush_counters(C, lane, k_events, k_commits, k_applied, k_msgs, k_dropped, k_elect, k_fatal);
    flush_ref_counters(C, lane, k_ref);
#ifdef RA_WARP_TIMELINE
    const u64 tl_g3 = tl_gtime(), tl_c3 = clock64();
    __syncwarp();
    if (lane == 0 && wtile < TL_WARPS_MAX) {
        u64* o = &g_tl[(size_t)wtile * TL_WORDS];
        for (int i = 10; i < TL_WORDS; i++) o[i] = tl_acc[warp][i];
        o[0] = tl_smid() | ((u64)tl_lead << 32) | (1ull << 63); o[1] = wtile;
        o[2] = tl_g0; o[3] = tl_g1; o[4] = tl_g2; o[5] = tl_g3; o[6] = tl_c0; o[7] = tl_c1; o[8] = tl_c2; o[9] = tl_c3;
        o[14] = tl_t1 - tl_t0; o[15] = tl_t2 - tl_t1; o[16] = tl_t3 - tl_t2; o[17] = tl_t3 ? tl_c3 - tl_t3 : 0;
    }
#endif
}

#undef RA_STEP_MINB
