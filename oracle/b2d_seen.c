/*
 * ORACLE -- test infrastructure, NOT product code.
 *
 * Seen lines (DESIGN.md C20): which segs of a compiled scene own at least one column of a frame in the front-to-back
 * solid pass.  It includes the oracle rasteriser (b2d_oracle.c) for its scene binding, integer helpers and frame state,
 * and runs its walk and draw_seg's clip loop without drawing: a seg owns column x at the point where draw_seg lets the
 * column past its `scale < 1` test (x in the seg's column interval, the column's window still open, a scale >= 1).  The
 * clip windows are updated as draw_seg updates them, so the seen set is the one of the oracle's own frames.  Sprites,
 * masked middles and planes change no window and mark nothing.
 *
 * Build: gcc, the flags of oracle/build.py (see oracle/seen.py).
 */
#include "b2d_oracle.c"

/* draw_seg's column loop, clip windows only: owned[si] = 1 when the seg owns a column */
static void seen_seg(Frame *f, int si, uint8_t *owned) {
    const Scene *sc = f->sc;
    const int32_t *S = sc->segs + 16 * si;
    if (S[3] & SEG_INVALID) return;
    const int W = f->vw.W, H = f->vw.H;
    const int64_t F = f->vw.F, FY2 = f->vw.FY2;
    int64_t ax = f->tx[S[0]], az = f->tz[S[0]], bx = f->tx[S[1]], bz = f->tz[S[1]];
    int64_t dxs = bx - ax, dzs = bz - az;
    int64_t C = az * dxs - ax * dzs;
    if (C <= 0) return;
    int64_t Nx = 2 * az, Nc = az * (1 - W) - ax * F;
    int64_t Dx = -2 * dzs, Dc = dxs * F - dzs * (1 - W);
    int64_t lo = 0, hi = W - 1;
    constrain(&lo, &hi, Dc, Dx, 1);
    constrain(&lo, &hi, Nc, Nx, 0);
    constrain(&lo, &hi, Dc - Nc, Dx - Nx, 0);
    if (lo > hi) return;
    int64_t Dbound = (dxs < 0 ? -dxs : dxs) * F + (dzs < 0 ? -dzs : dzs) * W;
    int sh = bitlen64((uint64_t)Dbound) - 31; if (sh < 0) sh = 0;
    int64_t M = F * C;
    int shm = bitlen64((uint64_t)M) - 31;
    uint64_t Mn = shm >= 0 ? ((uint64_t)M >> shm) : ((uint64_t)M << (-shm));
    uint64_t Rm = ((uint64_t)1 << 62) / Mn; if (Rm > 0xFFFFFFFFull) Rm = 0xFFFFFFFFull;
    int e = 5 - sh + shm;
    int64_t Dmax = M >> 8;
    int64_t scale_cap = FY2 << 17;

    const int32_t *SF = sc->sectors + 8 * S[2];
    int32_t fc = SF[1];
    int two = S[3] & SEG_TWO_SIDED;
    int32_t otop = S[13], obot = S[14];

    for (int x = (int)lo; x <= (int)hi; x++) {
        int ct = f->ctop[x], cb = f->cbot[x];
        if (ct >= cb) continue;
        int64_t D = Dc + Dx * x;
        int64_t Dt = D >> sh;
        if (Dt < 1) continue;
        int64_t Dcl = D < Dmax ? D : Dmax;
        uint64_t Dn = (uint64_t)(Dcl >> sh);
        if (Dn < 1) continue;
        uint64_t P = (Dn * Rm) >> 32;
        uint64_t prod = (uint64_t)FY2 * P;
        int64_t scale;
        if (e >= 0) scale = e > 63 ? 0 : (int64_t)(prod >> e);
        else scale = (-e) >= 20 ? scale_cap : (int64_t)(prod << (-e));
        if (scale > scale_cap) scale = scale_cap;
        if (scale < 1) continue;
        owned[si] = 1;                                        /* C20: the seg owns column x */
        const int32_t yscale = scale < 0x7FFFFFFF ? (int32_t)scale : 0x7FFFFFFF;
        int yfc = yrow(f, fc, yscale);
        if (!two) {
            f->ctop[x] = H; f->cbot[x] = 0; f->open_cols--;
        } else {
            int yot = yrow(f, otop, yscale), yob = yrow(f, obot, yscale);
            int y1 = clamp32(yfc, ct, cb);
            int y2 = clamp32(yot, y1, cb);
            int y3 = clamp32(yob, y2, cb);
            if (y2 >= y3) { f->ctop[x] = H; f->cbot[x] = 0; f->open_cols--; }
            else { f->ctop[x] = y2; f->cbot[x] = y3; }
        }
    }
}

/* walk(): the same front-to-back order and stopping rules, without the sprites (they change no window) */
static void seen_walk(Frame *f, uint32_t child, int depth, uint8_t *owned) {
    const Scene *sc = f->sc;
    if (f->open_cols <= 0 || depth > 4096) return;
    if (child & LEAF) {
        uint32_t id = child & 0x7FFFFFFFu;
        if ((int)id >= sc->nss) return;
        const int32_t *ss = sc->ssectors + 4 * id;
        if (ss[2] < 0) return;
        for (int i = 0; i < ss[1]; i++) seen_seg(f, ss[0] + i, owned);
        return;
    }
    if ((int)child >= sc->nnodes) return;
    const int32_t *n = sc->nodes + 16 * child;
    int64_t sd = ((int64_t)f->pose.y - ((int64_t)n[1] << 16)) * n[2]
               - ((int64_t)f->pose.x - ((int64_t)n[0] << 16)) * n[3];
    int side = sd > 0 ? 1 : 0;
    seen_walk(f, (uint32_t)n[12 + side], depth + 1, owned);
    seen_walk(f, (uint32_t)n[12 + (side ^ 1)], depth + 1, owned);
}

/* owned: n x nsegs bytes, set to 1 for every seg that owns a column of frame i (the rest are left as they are) */
int b2o_seen(const uint8_t *scene_blob, const b2o_view *vw, const b2o_pose *poses, int n, uint8_t *owned) {
    Scene sc;
    if (scene_bind(&sc, scene_blob) != 0) return -1;
    if (vw->W < 1 || vw->H < 1 || vw->W > 4096 || vw->H > 2160 || vw->F < 2 || vw->FY2 < 2
        || vw->F > (1 << 18) || vw->FY2 > (1 << 18) || vw->W > 256 * vw->F) return -2;
    int32_t *scratch = (int32_t *)malloc((2 * (size_t)sc.nverts + 2 * (size_t)vw->W + 1) * sizeof(int32_t));
    if (!scratch) return -3;
    for (int i = 0; i < n; i++) {
        Frame f;
        memset(&f, 0, sizeof f);
        f.sc = &sc; f.vw = *vw; f.pose = poses[i];
        f.tx = scratch; f.tz = f.tx + sc.nverts;
        f.ctop = f.tz + sc.nverts; f.cbot = f.ctop + vw->W;
        b2o_sincos_q30(poses[i].angle, &f.cosq, &f.sinq);
        int64_t px8 = asr64(poses[i].x, 8), py8 = asr64(poses[i].y, 8);
        for (int v = 0; v < sc.nverts; v++) {
            int64_t dx = ((int64_t)sc.verts[2 * v] << 8) - px8;
            int64_t dy = ((int64_t)sc.verts[2 * v + 1] << 8) - py8;
            f.tx[v] = (int32_t)asr64(dx * f.sinq - dy * f.cosq, 30);
            f.tz[v] = (int32_t)asr64(dx * f.cosq + dy * f.sinq, 30);
        }
        for (int x = 0; x < vw->W; x++) { f.ctop[x] = 0; f.cbot[x] = vw->H; }
        f.open_cols = vw->W;
        seen_walk(&f, sc.hdr[H_ROOT], 0, owned + (size_t)sc.nsegs * i);
    }
    free(scratch);
    return 0;
}
