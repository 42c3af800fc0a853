// CPU harness of the register window the border walk's hot loops keep over a halo tile (TileWin, contour_walk.cuh) and of
// trace_segment's grouped point stores.  TEST INFRASTRUCTURE ONLY.  Compiled with g++ by tests/test_hostsim_walk_window.py into a
// shared object of its own in a temporary directory; it is not linked into libfiducials_b200.so.  It includes hostsim.cpp for the
// plane packing and the start search.
#include "hostsim.cpp"

extern "C" {

// ---- register window of the hot loops (TileWin) against HaloView::idx9 ---------------------------------------------
// Every start crack of the plane walks up to max_steps steps with the reference walker (walk_resume_dir, one step at a time)
// while two windows follow it, one entered from the start pixel and one from the start's (tile, row, column) as a start record
// holds them; after every step both must show HaloView::idx9 of the walker's pixel.  Returns the number of mismatches;
// out[0] = steps compared, out[1] = steps that left the 30 x 30 tile.
int hs_window_check(const uint8_t* plane, int W, int H, int max_steps, int64_t* out) {
    HostPlane hp;
    pack_plane(plane, W, H, hp);
    std::vector<Start> starts;
    find_starts(hp, starts);
    const WalkCtx ctx = hp.ctx();
    const uint32_t tpr = (uint32_t)hp.tpr;
    int bad = 0;
    out[0] = out[1] = 0;
    for (const Start& s : starts) {
        WalkState st;
        if (walk_init(ctx, s.x, s.y, s.is_right, &st) != WALK_CONTINUE) continue;
        TileWin wa, wb;
        wa.enter(ctx.plane.base, tpr, (uint32_t)s.x | ((uint32_t)s.y << 16));
        const int tx = s.x / FID_HALO_T, ty = s.y / FID_HALO_T;
        wb.enter_tile(ctx.plane.base, (uint32_t)(ty * hp.tpr + tx), (uint32_t)(s.y - FID_HALO_T * ty + 1), (uint32_t)(s.x - FID_HALO_T * tx + 1));
        if (wa.idx9() != ctx.plane.idx9(s.x, s.y) || wb.idx9() != wa.idx9()) bad++;
        for (int k = 0; k < max_steps; k++) {
            const int px = st.x, py = st.y;
            const int r = s.is_right ? walk_resume_dir<true>(ctx, s.x, s.y, 1 << 30, 1, &st) : walk_resume_dir<false>(ctx, s.x, s.y, 1 << 30, 1, &st);
            wa.step(ctx.plane.base, tpr, st.x - px, st.y - py);
            wb.step(ctx.plane.base, tpr, st.x - px, st.y - py);
            const uint32_t want = ctx.plane.idx9(st.x, st.y);
            if (wa.idx9() != want || wb.idx9() != want) bad++;
            out[0]++;
            if (st.x / FID_HALO_T != px / FID_HALO_T || st.y / FID_HALO_T != py / FID_HALO_T) out[1]++;
            if (r != WALK_CONTINUE) break;
        }
    }
    return bad;
}

// Every segment of every contour of the plane (checkpoints every ck_step steps), traced on its own into a sentinel-filled buffer
// with the chain placed at word offsets 4 .. 7: the segment's words must be the contour's points as trace_forward writes them and
// no other word may change.  Returns the number of wrong words; out[0] = segments traced, out[1] = backward segments among them,
// out[2 + (off & 3)] = segments whose first word sat at that alignment.
int hs_trace_segment_check(const uint8_t* plane, int W, int H, int ck_step, int64_t* out) {
    HostPlane hp;
    pack_plane(plane, W, H, hp);
    std::vector<Start> starts;
    find_starts(hp, starts);
    const WalkCtx ctx = hp.ctx();
    int bad = 0;
    for (int k = 0; k < 6; k++) out[k] = 0;
    const uint32_t sentinel = 0xFFFFFFFFu;
    for (const Start& s : starts) {
        WalkState st;
        if (walk_init(ctx, s.x, s.y, s.is_right, &st) != WALK_CONTINUE) continue;
        WalkState2 s2;
        if (s.is_right) walk_split<true>(s.x, s.y, st, &s2); else walk_split<false>(s.x, s.y, st, &s2);
        WalkCkpt ck;
        ck.count[0] = ck.count[1] = 0;
        int last_f = 0, last_b = 0, r = WALK_CONTINUE;
        while (r == WALK_CONTINUE) {
            r = s.is_right ? walk_resume_bidir<true>(ctx, s.x, s.y, 1 << 30, 2, &s2) : walk_resume_bidir<false>(ctx, s.x, s.y, 1 << 30, 2, &s2);
            if (r == WALK_CONTINUE) walk_checkpoint(s2, &ck, &last_f, &last_b, ck_step);
        }
        if (r != WALK_CANONICAL) continue;
        const int n = s2.n;
        std::vector<Pt16> ref((size_t)((n + 3) & ~3));
        trace_forward(ctx, s.x, s.y, s.is_right, n, ref.data());
        for (uint32_t chain_off = 4; chain_off < 8; chain_off++) {
            std::vector<SegRec> segs((size_t)segment_count(&ck));
            make_segments(ctx, s.x, s.y, s.is_right, n, s2.nf, &ck, 0u, chain_off, [&](int k, const SegRec& sr) { segs[(size_t)k] = sr; });
            for (const SegRec& sr : segs) {
                std::vector<uint32_t> buf((size_t)n + 16, sentinel);
                trace_segment(ctx, sr, buf.data());
                const int count = (int)(sr.dn >> 3), backward = (int)(sr.meta & 1u);
                const int lo = backward ? (int)sr.off - count : (int)sr.off, hi = lo + count;  // the segment's words
                for (int w = 0; w < (int)buf.size(); w++) {
                    uint32_t want = sentinel;
                    if (w >= lo && w < hi) {
                        const Pt16& p = ref[(size_t)(w - (int)chain_off)];
                        want = (uint32_t)(uint16_t)p.x | ((uint32_t)(uint16_t)p.y << 16);
                    }
                    if (buf[(size_t)w] != want) bad++;
                }
                out[0]++;
                out[1] += backward;
                out[2 + ((backward ? sr.off - 1u : sr.off) & 3u)]++;
            }
        }
    }
    return bad;
}

}  // extern "C"
