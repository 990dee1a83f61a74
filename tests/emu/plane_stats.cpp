/* TEST INFRASTRUCTURE -- not part of the product.
 *
 * The host emulation (ra_emu.cpp, compiled into this one translation unit unchanged) built with RA_PLANE_STATS:
 * every record the device logic stores into a record plane is counted by type and form, and the record-plane codec
 * is exposed through both index widths.  tests/emu_lib.py (stats_lib) compiles this file on its own (g++, into a
 * temporary directory) and loads it next to the regular emulation library; both export the same names, so it
 * is linked -Bsymbolic and loaded RTLD_LOCAL (ctypes' default).
 */
#define RA_PLANE_STATS 1
#include "ra_emu.cpp"

/* records stored into a plane since the last reset, by type (0..15) and form (0 short, 1 head, 3 long) */
static unsigned long long g_plane_forms[16][4];
extern "C" void ra_emu_plane_store(unsigned type, unsigned form)
{ __atomic_fetch_add(&g_plane_forms[type & 15u][form & 3u], 1ull, __ATOMIC_RELAXED); }
extern "C" void ra_emu_plane_forms(unsigned long long* out64, int reset)
{
    memcpy(out64, g_plane_forms, sizeof g_plane_forms);
    if (reset) memset(g_plane_forms, 0, sizeof g_plane_forms);
}

/* One ABI record through both passes, with the tile pre-filled with `fill` bytes (what a staging slot holds from an
 * earlier tile):
 *   wide    st_rec_plane -> ld_rec_plane                                          -> out_wide
 *   narrow  the stored chunks -> ra_narrow::rec_decode (*narrow_fits: every field < 2^30); when it fits, the narrow
 *           record -> ra_narrow::st_rec_plane into a second tile -> ld_rec_plane   -> out_narrow
 * *form: what the wide store wrote (0 short, RF_NOT_SHORT head, | RF_TAIL long); *form_narrow: the narrow store. */
extern "C" int ra_emu_codec_roundtrip2(const ra_event* in, int fill, ra_event* out_wide, int* form,
                                       ra_event* out_narrow, int* narrow_fits, int* form_narrow)
{
    if (!in || !out_wide || !out_narrow || !form || !narrow_fits || !form_narrow) return RA_E_INVAL;
    static thread_local ulonglong2 plane[4 * RT], plane2[4 * RT];
    memset(plane, fill, sizeof plane); memset(plane2, fill ^ 0x5A, sizeof plane2);
    const u32 row = in->row & (RT - 1);
    *form = (int)st_rec_plane(plane, 1, 0, row, ld_rec(in));
    st_rec(out_wide, ld_rec_plane(plane, 1, 0, row));
    const ulonglong2* q = plane + rec_word(1, 0, row, 0);
    ra_narrow::Rec e;
    *narrow_fits = ra_narrow::rec_decode(q[0], q[RT], q[2 * RT], q[3 * RT], row, e) ? 1 : 0;
    memset(out_narrow, 0, sizeof *out_narrow);
    *form_narrow = -1;
    if (*narrow_fits) {
        *form_narrow = (int)ra_narrow::st_rec_plane(plane2, 1, 0, row, e);
        st_rec(out_narrow, ld_rec_plane(plane2, 1, 0, row));
    }
    return RA_OK;
}
