// host_flood.cu -- a HOST-side caller of the public C ABI (ra_engine_step with host buffers).
//
// It plays the part of the Erlang side in the benchmark: per step it hands the engine the
// events only the host can produce -- {ra_log_event,{written,..}} for every WAL_APPEND note of
// the previous step (ra_log_wal.erl:784-808), one {commands,_} per leader (the ra_bench-style
// client flood, src/ra_bench.erl:89-136) and election_timeout when a member heard no leader
// for a while (ra_server_proc.erl:1927-1946) -- and reads the notes back.  Everything goes
// through ra_engine_step: H2D of the events, D2H of the notes, every step.
#include <chrono>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <omp.h>
#include <vector>
#ifndef RA_NO_CUDA
#include <cuda_runtime.h>
#endif
#include "../../include/ra_engine.h"

typedef unsigned long long u64;
typedef unsigned int u32;

static inline u64 mix64(u64 x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// one engine of the simulation = one partition of the groups, with its own pinned batch / note buffers
struct Part {
    ra_engine* e;
    u32 groups, members, rows;
    std::vector<unsigned char> role, idle;
    ra_host_event* ev;  size_t ev_cap; // pinned; the flood only has host-origin events: 32-byte records
    ra_event* msgs; size_t msgs_cap;  // pinned
    ra_note* notes; size_t notes_cap; // pinned
    size_t n_ev;
    u64 step;
    u64 seed_off;                     // partition p runs the model with seed + p (independent groups)
    std::vector<uint64_t> last_c;     // compact note stream: the decoder's per-row state
    size_t n_ext;                     // extension entries of the call collected last
};

// a driver = one host thread that owns some of the partitions (collect, model, submit, round robin) and a team of
// model threads.  One driver is the default; RA_HOSTSIM_DRIVERS=2 lets one's waits overlap the other's model
struct Driver {
    u32 threads;
    std::vector<std::vector<ra_host_event>> tmp;
    std::vector<size_t> cnt, off;
    double t_model, t_step;
    u64 h2d, d2h, calls;
    int rc;
};

struct ra_hostsim {
    std::vector<Part> parts;
    u32 threads;                     // model threads in total
    int compact;                     // notes travel as 16-byte units (RA_HOSTSIM_COMPACT, default on)
    std::vector<Driver> drivers;
    double t_model, t_step;          // seconds spent in the host model / waiting inside engine calls (max over drivers)
    u64 h2d, d2h, calls; double seconds;
};

#ifndef RA_NO_CUDA
extern "C" void* ra_engine_alloc_host(size_t bytes)
{
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void ra_engine_free_host(void* p) { if (p) cudaFreeHost(p); }
#else   /* tests/emu: this caller over the host emulation of the engine, plain host memory */
extern "C" void* ra_engine_alloc_host(size_t bytes) { return malloc(bytes ? bytes : 16); }
extern "C" void ra_engine_free_host(void* p) { free(p); }
#endif

extern "C" void ra_hostsim_destroy(ra_hostsim* s)
{
    if (!s) return;
    for (Part& p : s->parts) { ra_engine_free_host(p.ev); ra_engine_free_host(p.msgs); ra_engine_free_host(p.notes); }
    delete s;
}

// K engines holding disjoint sets of groups, driven by ONE host thread through ra_engine_submit_host /
// ra_engine_collect: while the notes of one partition travel to the host and its model runs, the batch of
// another travels to the device and its kernels run (PCIe is full duplex).
extern "C" int ra_hostsim_create_multi(ra_engine* const* engines, uint32_t n, ra_hostsim** out)
{
    if (!engines || !n || !out) return RA_E_INVAL;
    ra_hostsim* s = new ra_hostsim();
    s->parts.resize(n);
    u32 max_rows = 0;
    for (u32 i = 0; i < n; i++) {
        Part& p = s->parts[i];
        ra_engine_cfg cfg;
        if (!engines[i] || ra_engine_get_cfg(engines[i], &cfg) != RA_OK || !cfg.route_on_device) { ra_hostsim_destroy(s); return RA_E_INVAL; }
        p.e = engines[i]; p.groups = cfg.n_groups; p.members = cfg.n_members; p.rows = p.groups * p.members;
        p.role.assign(p.rows, RA_FOLLOWER); p.idle.assign(p.rows, 0);
        // a flood row emits <= 2 WAL_APPEND + COMMIT + APPLY + STATUS notes per step in steady state; the rare
        // step that needs more is fetched again with a bigger buffer (RA_E_CAPACITY loses nothing)
        p.ev_cap = (size_t)p.rows * RA_LOCAL_CAP; p.msgs_cap = 1024; p.notes_cap = (size_t)p.rows * 6;
        p.ev = (ra_host_event*)ra_engine_alloc_host(p.ev_cap * sizeof(ra_host_event));
        p.msgs = (ra_event*)ra_engine_alloc_host(p.msgs_cap * sizeof(ra_event));
        p.notes = (ra_note*)ra_engine_alloc_host(p.notes_cap * sizeof(ra_note));
        if (!p.ev || !p.msgs || !p.notes) { ra_hostsim_destroy(s); return RA_E_NOMEM; }
        p.n_ev = 0; p.step = 0; p.seed_off = i; p.n_ext = 0;
        if (p.rows > max_rows) max_rows = p.rows;
    }
    {
        unsigned hc = std::thread::hardware_concurrency();
        const char* env = getenv("RA_HOSTSIM_THREADS");
        s->threads = env ? (u32)atoi(env) : (hc > 16 ? 16u : (hc ? hc : 1u));
        if (s->threads < 1) s->threads = 1;
        const char* de = getenv("RA_HOSTSIM_DRIVERS");
        u32 nd = de ? (u32)atoi(de) : 1u;      // one driver: the host model's threads, not the driver's waits, bound the flood
        if (nd < 1) nd = 1;
        if (nd > n) nd = n;
        s->drivers.resize(nd);
        for (Driver& d : s->drivers) {
            d.threads = s->threads / nd ? s->threads / nd : 1;
            d.tmp.resize(d.threads);
            d.cnt.assign(d.threads, 0); d.off.assign(d.threads + 1, 0);
        }
    }
    {   // notes as 16-byte units (half the device->host bytes of a step) unless RA_HOSTSIM_COMPACT=0
        const char* ce = getenv("RA_HOSTSIM_COMPACT");
        s->compact = !(ce && ce[0] == '0');
#ifdef RA_NO_CUDA
        s->compact = 0;                              // (the host emulation of tests/emu/ has the plain format only)
#else
        if (s->compact)
            for (Part& p : s->parts) {
                if (ra_engine_set_note_format(p.e, 1) != RA_OK) { s->compact = 0; break; }
                p.last_c.assign(p.rows, 0);
            }
        if (!s->compact) for (Part& p : s->parts) { ra_engine_set_note_format(p.e, 0); p.last_c.clear(); }
#endif
    }
    s->h2d = s->d2h = s->calls = 0; s->seconds = 0; s->t_model = s->t_step = 0;
    *out = s;
    return RA_OK;
}

extern "C" int ra_hostsim_create(ra_engine* e, ra_hostsim** out) { return ra_hostsim_create_multi(&e, 1, out); }

static inline void put(ra_host_event* e, u32 row, u32 type, u32 n, u64 term, u64 a, u64 b)
{
    e->row = row; e->type = (uint8_t)type; e->flags = 0; e->n = (uint16_t)n; e->term = term; e->a = a; e->b = b;
}
static inline void put(ra_event* e, u32 row, u32 type, u32 n, u64 term, u64 a, u64 b)
{
    memset(e, 0, sizeof *e);
    e->row = row; e->type = (uint8_t)type; e->from_slot = RA_NO_SLOT; e->n = (uint16_t)n;
    e->term = term; e->a = a; e->b = b;
}

// notes of one step -> events of the next (the flood host model, DESIGN.md), rows [r0, r1) of one partition
// note16_decode is defined below (compact note stream)
static inline void note16_decode(const ra_note16* units, size_t n_notes, size_t i, uint64_t* last_wal_c, ra_note* o);

template <bool COMPACT>
static size_t model_range(Part* s, const ra_note* notes, size_t n_notes, u32 r0, u32 r1, ra_host_event* out,
                          u32 cmds, u32 permille, u64 seed, bool run_model)
{
    const ra_note16* units = reinterpret_cast<const ra_note16*>(notes);      // COMPACT: 16-byte units, extensions behind
    auto row_at = [&](size_t k) -> u32 { return COMPACT ? units[k].row : notes[k].row; };
    // first note of row r0 (notes are ordered by row)
    size_t lo = 0, hi = n_notes;
    while (lo < hi) { size_t mid = (lo + hi) / 2; if (row_at(mid) < r0) lo = mid + 1; else hi = mid; }
    size_t ne = 0, i = lo;
    for (u32 row = r0; row < r1; row++) {
        ra_note wa, wb, cur;                                 // the row's last two WAL_APPEND notes, the note at hand
        const ra_note* w0 = nullptr; const ra_note* w1 = nullptr;
        u32 status = 0; bool fatal = false;
        const ra_note* last = nullptr;
        for (; i < n_notes && row_at(i) == row; i++) {
            if (COMPACT) note16_decode(units, n_notes, i, s->last_c.data(), &cur);
            const ra_note& n = COMPACT ? cur : notes[i];
            last = &n;
            if (n.type == RA_NOTE_WAL_APPEND) {
                if (w1) { wa = *w1; w0 = &wa; }
                wb = n; w1 = &wb;
            }
            else if (n.type == RA_NOTE_STATUS) {
                status = n.aux;
                s->role[row] = (unsigned char)((n.b >> 24) & 0xff);
                if (n.aux & RA_ST_FATAL) fatal = true;
            }
        }
        if (last && last->type != RA_NOTE_STATUS) status |= last->aux;   // flags riding in the last note
        if (!run_model || fatal) continue;
        if (w0) put(&out[ne++], row, RA_EV_WRITTEN, 0, w0->c, w0->a, w0->b);
        if (w1) put(&out[ne++], row, RA_EV_WRITTEN, 0, w1->c, w1->a, w1->b);
        const u32 role = s->role[row];
        if (role == RA_LEADER && cmds) put(&out[ne++], row, RA_EV_COMMAND, cmds, 0, 0, 0);
        u32 idle = s->idle[row];
        if (role == RA_LEADER || (status & RA_ST_LEADER_MSG)) idle = 0;
        else if (idle < 15) idle++;
        bool fire = false;
        if (role != RA_LEADER) {
            const u32 group = row % s->groups, slot = row / s->groups;
            u32 h = (u32)(mix64(seed ^ (s->step * 0x9E3779B97F4A7C15ull) ^ ((u64)group * 0xD1B54A32D192ED03ull)) >> 32);
            if (permille && (h % 1000u) < permille && ((h / 1000u) % s->members) == slot) fire = true;
            if (idle >= 8) {                                // the second hash only matters from 8 idle steps on
                const u32 h2 = (u32)(mix64(seed ^ ((u64)row * 0xA24BAED4963EE407ull) ^ s->step) >> 32);
                if (idle >= 8 + (h2 & 7u)) fire = true;
            }
        }
        if (fire) { put(&out[ne++], row, RA_EV_ELECTION_TIMEOUT, 0, 0, 0, 0); idle = 0; }
        s->idle[row] = (unsigned char)idle;
    }
    return ne;
}

// the model over all rows of a partition on s->threads host threads (OpenMP keeps the team alive between
// steps): each thread fills a private buffer for its row range, then the pieces are copied, in row order, into
// the partition's pinned batch
static void model(Driver* s, Part* p, size_t n_notes, u32 cmds, u32 permille, u64 seed, bool run_model)
{
    const int T = (int)s->threads;
    const bool compact = !p->last_c.empty();
    if (T <= 1 || p->rows < 4096) {
        p->n_ev = compact ? model_range<true>(p, p->notes, n_notes, 0, p->rows, p->ev, cmds, permille, seed, run_model)
                          : model_range<false>(p, p->notes, n_notes, 0, p->rows, p->ev, cmds, permille, seed, run_model);
        return;
    }
    std::vector<size_t>& cnt = s->cnt;
    std::vector<size_t>& off = s->off;
#pragma omp parallel num_threads(T)
    {
        const int t = omp_get_thread_num();
        const u32 r0 = (u32)((u64)p->rows * t / T), r1 = (u32)((u64)p->rows * (t + 1) / T);
        if (s->tmp[t].size() < (size_t)(r1 - r0) * RA_LOCAL_CAP) s->tmp[t].resize((size_t)(r1 - r0) * RA_LOCAL_CAP);
        cnt[t] = compact ? model_range<true>(p, p->notes, n_notes, r0, r1, s->tmp[t].data(), cmds, permille, seed, run_model)
                         : model_range<false>(p, p->notes, n_notes, r0, r1, s->tmp[t].data(), cmds, permille, seed, run_model);
#pragma omp barrier
#pragma omp single
        {
            off[0] = 0;
            for (int k = 0; k < T; k++) off[k + 1] = off[k] + cnt[k];
        }
        if (cnt[t]) memcpy(p->ev + off[t], s->tmp[t].data(), cnt[t] * sizeof(ra_host_event));
    }
    p->n_ev = off[T];
}

// capacity of a partition's note buffer in the units of its note format (a 32-byte slot holds two 16-byte units)
static inline size_t note_cap_of(const Part& p) { return p.last_c.empty() ? p.notes_cap : 2 * p.notes_cap; }

// collect a partition's call; a note buffer that turned out too small is grown and the outputs fetched again
static int collect_part(Driver* s, Part* p, size_t* nn)
{
    size_t nm = 0;
    int rc = ra_engine_collect(p->e, &nm, nn);
#ifndef RA_NO_CUDA
    if (rc == RA_E_CAPACITY) {
        if (*nn + *nn / 8 > p->notes_cap || !p->last_c.empty()) {   // (compact: the extension count is not known here)
            ra_engine_free_host(p->notes);
            p->notes_cap = *nn * 2 + 1024;
            p->notes = (ra_note*)ra_engine_alloc_host(p->notes_cap * sizeof(ra_note));
        }
        if (nm > p->msgs_cap) {
            ra_engine_free_host(p->msgs);
            p->msgs_cap = nm + nm / 4;
            p->msgs = (ra_event*)ra_engine_alloc_host(p->msgs_cap * sizeof(ra_event));
        }
        if (!p->notes || !p->msgs) return RA_E_NOMEM;
        rc = ra_engine_fetch_output(p->e, p->msgs, p->msgs_cap, &nm, p->notes, note_cap_of(*p), nn);
    }
#endif
    if (rc) return rc;
#ifndef RA_NO_CUDA
    if (!p->last_c.empty()) {
        p->n_ext = ra_engine_last_ext_count(p->e);
        s->d2h += (*nn + 2 * p->n_ext) * sizeof(ra_note16) + nm * sizeof(ra_event);
        return RA_OK;
    }
#endif
    s->d2h += *nn * sizeof(ra_note) + nm * sizeof(ra_event);
    return RA_OK;
}

// the partitions i with i % n_drivers == k, driven by one thread
static void drive(ra_hostsim* s, u32 k, uint32_t n_steps, uint32_t cmds, uint32_t permille, uint64_t seed, int bootstrap)
{
    Driver* d = &s->drivers[k];
    const size_t P = s->parts.size(), D = s->drivers.size();
    d->h2d = d->d2h = d->calls = 0; d->t_model = d->t_step = 0; d->rc = RA_OK;
    size_t nn = 0;
    int rc;
#define FAIL_IF(x) do { if ((rc = (x))) { d->rc = rc; return; } } while (0)
    if (bootstrap) {
        for (size_t i = k; i < P; i += D) {
            Part& p = s->parts[i];
            for (u32 g = 0; g < p.groups; g++) put(&p.ev[g], g, RA_EV_ELECTION_TIMEOUT, 0, 0, 0, 0);
            FAIL_IF(ra_engine_submit_host(p.e, p.ev, p.groups, p.msgs, p.msgs_cap, p.notes, note_cap_of(p)));
            d->h2d += (u64)p.groups * sizeof(ra_host_event); d->calls++;
        }
        for (size_t i = k; i < P; i += D) {
            Part& p = s->parts[i];
            FAIL_IF(collect_part(d, &p, &nn));
            model(d, &p, nn, cmds, permille, seed + p.seed_off, false);   // roles only; no model run for this step
            p.n_ev = 0;
        }
    }
    if (!n_steps) return;
    // software pipeline over the partitions: every partition always has one call in flight
    for (size_t i = k; i < P; i += D) {
        Part& p = s->parts[i];
        FAIL_IF(ra_engine_submit_host(p.e, p.ev, p.n_ev, p.msgs, p.msgs_cap, p.notes, note_cap_of(p)));
        d->h2d += (u64)p.n_ev * sizeof(ra_host_event); d->calls++;
    }
    for (u32 t = 0; t < n_steps; t++) {
        for (size_t i = k; i < P; i += D) {
            Part& p = s->parts[i];
            auto a0 = std::chrono::steady_clock::now();
            FAIL_IF(collect_part(d, &p, &nn));
            auto a1 = std::chrono::steady_clock::now();
            model(d, &p, nn, cmds, permille, seed + p.seed_off, true);
            p.step++;
            auto a2 = std::chrono::steady_clock::now();
            if (t + 1 < n_steps) {
                FAIL_IF(ra_engine_submit_host(p.e, p.ev, p.n_ev, p.msgs, p.msgs_cap, p.notes, note_cap_of(p)));
                d->h2d += (u64)p.n_ev * sizeof(ra_host_event); d->calls++;
            }
            auto a3 = std::chrono::steady_clock::now();
            d->t_step += std::chrono::duration<double>(a1 - a0).count() + std::chrono::duration<double>(a3 - a2).count();
            d->t_model += std::chrono::duration<double>(a2 - a1).count();
        }
    }
#undef FAIL_IF
}

extern "C" int ra_hostsim_run(ra_hostsim* s, uint32_t n_steps, uint32_t cmds, uint32_t permille,
                              uint64_t seed, int bootstrap)
{
    if (!s) return RA_E_INVAL;
    auto t0 = std::chrono::steady_clock::now();
    const u32 D = (u32)s->drivers.size();
    if (D == 1) drive(s, 0, n_steps, cmds, permille, seed, bootstrap);
    else {
        std::vector<std::thread> th;
        for (u32 k = 0; k < D; k++) th.emplace_back(drive, s, k, n_steps, cmds, permille, seed, bootstrap);
        for (auto& t : th) t.join();
    }
    s->h2d = s->d2h = s->calls = 0; s->t_model = s->t_step = 0;
    int rc = RA_OK;
    for (Driver& d : s->drivers) {
        s->h2d += d.h2d; s->d2h += d.d2h; s->calls += d.calls;
        if (d.t_model > s->t_model) s->t_model = d.t_model;
        if (d.t_step > s->t_step) s->t_step = d.t_step;
        if (d.rc && !rc) rc = d.rc;
    }
    s->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

extern "C" int ra_hostsim_stats(ra_hostsim* s, uint64_t* h2d, uint64_t* d2h, double* seconds, uint64_t* calls)
{
    if (!s) return RA_E_INVAL;
    if (h2d) *h2d = s->h2d; if (d2h) *d2h = s->d2h; if (seconds) *seconds = s->seconds; if (calls) *calls = s->calls;
    return RA_OK;
}

/* where the wall time of the last run went: waiting inside engine calls vs in the host model */
extern "C" int ra_hostsim_breakdown(ra_hostsim* s, double* step_seconds, double* model_seconds)
{
    if (!s) return RA_E_INVAL;
    if (step_seconds) *step_seconds = s->t_step; if (model_seconds) *model_seconds = s->t_model;
    return RA_OK;
}


// ---- compact note stream: the decoder (include/ra_engine.h, ra_note16) ------------------------------------
static inline void note16_decode(const ra_note16* units, size_t n_notes, size_t i, uint64_t* last_wal_c, ra_note* o)
{
    const ra_note16& u = units[i];
    o->row = u.row; o->type = (uint8_t)(u.type & 0x3fu); o->aux = u.aux;
    if (u.type & RA_N16_EXT) {
        const uint64_t* x = reinterpret_cast<const uint64_t*>(units + n_notes + 2 * (size_t)u.a);
        o->slot = u.n; o->a = x[0]; o->b = x[1]; o->c = x[2];
    } else {
        o->slot = 0; o->a = u.a; o->b = u.a + u.n;
        o->c = (u.type & RA_N16_SAME_TERM) ? last_wal_c[u.row] : 0;
    }
    if (o->type == RA_NOTE_WAL_APPEND) last_wal_c[u.row] = o->c;
}

extern "C" size_t ra_notes16_expand(const ra_note16* units, size_t n_notes, size_t n_ext, uint64_t* last_wal_c,
                                    ra_note* out, size_t cap)
{
    (void)n_ext;
    if (!units || !out || !last_wal_c || cap < n_notes) return 0;
    for (size_t i = 0; i < n_notes; i++) note16_decode(units, n_notes, i, last_wal_c, &out[i]);
    return n_notes;
}

// ---- written-event source: one WAL batch -> one grouped event array (include/ra_engine.h) -----------
// Within one call a row gets at most max_per_row records and every row's records are adjacent; a writer
// whose ranges do not fit stops the call there (its remaining ranges must not be reordered behind other
// rows of a later call, and a second run of the same row in one batch would break the grouping contract).
extern "C" size_t ra_wal_batch_to_events(const ra_wal_writer* w, size_t n, uint32_t max_per_row,
                                         ra_event* out, size_t cap, ra_wal_resume* resume)
{
    if (!w || !out || !resume || max_per_row == 0 || max_per_row > RA_LOCAL_CAP) return 0;
    size_t ne = 0;
    u32 wi = resume->writer, ri = resume->range;
    u32 run_row = 0xFFFFFFFFu, taken = 0;           // records of the current run of one row (a writer that
    while (wi < n) {                                // changed term mid-batch is notified twice, back to back)
        const ra_wal_writer& x = w[wi];
        if (x.row != run_row) { run_row = x.row; taken = 0; }
        while (ri < x.n_ranges && taken < max_per_row && ne < cap) {
            put(&out[ne++], x.row, RA_EV_WRITTEN, 0, x.term, x.ranges[2 * ri], x.ranges[2 * ri + 1]);
            ri++; taken++;
        }
        if (ri < x.n_ranges) break;                 // out of room for this row (or for the batch): resume here
        wi++; ri = 0;
        if (ne >= cap) break;
    }
    resume->writer = wi; resume->range = ri;
    return ne;
}
