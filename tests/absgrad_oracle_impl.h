/*
 * absgrad_oracle_impl.h — the absolute-gradient statistic (DGR_RASTER_ABS_GRAD) on the C oracle's forward state, hand-derived.
 * Included twice by absgrad_oracle.c (REAL=float, SUF=f32 and REAL=double, SUF=f64) after the oracle itself.
 *
 * The per-pixel loop is the oracle's backward loop (oracle/dgr_oracle_impl.h, dgr_oracle_backward): same traversal, skip rules and
 * dL/dalpha recurrence.  Where that loop adds the pixel's term of dL/dmean_px into a sum, this one also adds its absolute value:
 * out[4g + 0..3] = sum |t_x|, sum |t_y|, sum t_x, sum t_y over the pixels g is evaluated at, t = the pixel's term of dL/dmean_px in
 * pixel units (double accumulators, serial: the order is fixed).
 */
void FN(dgr_oracle_absgrad)(const FN(Ctx) *c, const REAL *gC, const REAL *gD, const REAL *gA, double *out)
{
    const int P = c->P, H = c->H, W = c->W, gx = c->gx, gy = c->gy;
    const size_t HW = (size_t)H * W;
    memset(out, 0, (size_t)(P > 0 ? P : 1) * 4 * sizeof(double));
    for (int tile = 0; tile < gx * gy; tile++) {
        int tx0 = (tile % gx) * DGR_TILE, ty0 = (tile / gx) * DGR_TILE;
        unsigned s = c->ranges[2 * tile];
        for (int yy = ty0; yy < ty0 + DGR_TILE && yy < H; yy++) for (int xx = tx0; xx < tx0 + DGR_TILE && xx < W; xx++) {
            size_t pix = (size_t)yy * W + xx;
            unsigned last = c->n_contrib[pix];
            REAL gc[3] = { gC ? gC[pix] : 0, gC ? gC[HW + pix] : 0, gC ? gC[2 * HW + pix] : 0 };
            REAL gd = gD ? gD[pix] : 0, ga = gA ? gA[pix] : 0;
            REAL T_final = c->final_T[pix], T = T_final;
            REAL accC[3] = { 0, 0, 0 }, accD = 0, accA = 0, la = 0, lc[3] = { 0, 0, 0 }, ld = 0;
            REAL bgdot = c->bg[0] * gc[0] + c->bg[1] * gc[1] + c->bg[2] * gc[2];
            for (unsigned k = last; k-- > 0;) {
                unsigned g = c->point_list[s + k];
                REAL dx = c->px[g] - (REAL)xx, dy = c->py[g] - (REAL)yy;
                const REAL *co = c->conic + 3 * (size_t)g;
                REAL power = (REAL)-0.5 * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                if (power > 0) continue;
                REAL G = (REAL)exp((double)power);
                REAL a = FN(rmin)((REAL)DGR_ALPHA_MAX, c->opac[g] * G);
                if (a < (REAL)DGR_ALPHA_MIN) continue;
                T = T / ((REAL)1 - a);
                REAL dL_da = 0;
                for (int ch = 0; ch < 3; ch++) {
                    accC[ch] = la * lc[ch] + ((REAL)1 - la) * accC[ch]; lc[ch] = c->rgb[3 * (size_t)g + ch];
                    dL_da += (lc[ch] - accC[ch]) * gc[ch];
                }
                accD = la * ld + ((REAL)1 - la) * accD; ld = c->depth[g];
                dL_da += (ld - accD) * gd;
                accA = la + ((REAL)1 - la) * accA;
                dL_da += ((REAL)1 - accA) * ga;
                dL_da *= T;
                dL_da += (-T_final / ((REAL)1 - a)) * bgdot;
                la = a;
                REAL dL_dG = c->opac[g] * dL_da;            /* min(0.99, .) straight-through, as the backward */
                REAL gdx = co[0] * dx + co[1] * dy, gdy = co[2] * dy + co[1] * dx;
                double tx = (double)(dL_dG * -G * gdx), ty = (double)(dL_dG * -G * gdy);
                double *o = out + 4 * (size_t)g;
                o[0] += fabs(tx); o[1] += fabs(ty); o[2] += tx; o[3] += ty;
            }
        }
    }
}
