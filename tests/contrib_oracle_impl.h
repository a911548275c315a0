/*
 * contrib_oracle_impl.h — the blending-weight statistics (DGR_RASTER_CONTRIB) on the C oracle's forward state.
 * Included twice by contrib_oracle.c (REAL=float, SUF=f32 and REAL=double, SUF=f64) after the oracle itself.
 *
 * The per-pixel loop is the oracle's forward compositing (oracle/dgr_oracle_impl.h, dgr_oracle_forward): same list, skip rules
 * and transmittance recurrence, walked up to the pixel's last composited record (n_contrib).  Every composited (pixel, Gaussian)
 * pair adds w = alpha T to out[2g] and raises out[2g + 1] (double accumulators, serial: the order is fixed).
 */
void FN(dgr_oracle_contrib)(const FN(Ctx) *c, double *out)
{
    const int P = c->P, H = c->H, W = c->W, gx = c->gx, gy = c->gy;
    memset(out, 0, (size_t)(P > 0 ? P : 1) * 2 * sizeof(double));
    for (int tile = 0; tile < gx * gy; tile++) {
        int tx0 = (tile % gx) * DGR_TILE, ty0 = (tile / gx) * DGR_TILE;
        unsigned s = c->ranges[2 * tile];
        for (int yy = ty0; yy < ty0 + DGR_TILE && yy < H; yy++) for (int xx = tx0; xx < tx0 + DGR_TILE && xx < W; xx++) {
            size_t pix = (size_t)yy * W + xx;
            unsigned last = c->n_contrib[pix];
            REAL T = 1;
            for (unsigned k = 0; k < last; k++) {
                unsigned g = c->point_list[s + k];
                REAL dx = c->px[g] - (REAL)xx, dy = c->py[g] - (REAL)yy;
                const REAL *co = c->conic + 3 * (size_t)g;
                REAL power = (REAL)-0.5 * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                if (power > 0) continue;
                REAL a = FN(rmin)((REAL)DGR_ALPHA_MAX, c->opac[g] * (REAL)exp((double)power));
                if (a < (REAL)DGR_ALPHA_MIN) continue;
                REAL w = a * T;
                double *o = out + 2 * (size_t)g;
                o[0] += (double)w;
                if ((double)w > o[1]) o[1] = (double)w;
                T = T * ((REAL)1 - a);
            }
        }
    }
}
