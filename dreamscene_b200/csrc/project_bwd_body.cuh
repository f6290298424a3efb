// The statements of project_bwd_kernel, project_bwd_stats_kernel and project_bwd_rows_frozen_kernel (project.cu),
// included into the body of each.  In scope: the kernel's parameters and the compile-time MT, RAW, DYN, FROZEN, STATS
// and LIVE (see those kernels).
extern __shared__ __align__(16) float sh_buf[];
__shared__ uint8_t vis_s[kBlock];
const ViewNoise nz = view_noise<DYN>(sc, p);
// this launch covers Gaussians [g_base, g_end) (the whole range, or one chunk when the host
// overlaps the gradient all-reduce of finished chunks with the remaining ones)
const int g0 = g_base + blockIdx.x * kBlock;
const int i = g0 + threadIdx.x;
const bool active = i < g_end;
const bool fz = frozen_row<FROZEN>(sc, active, i);
const bool vis = active && !fz && (__ldg(radii + rec_base + i) > 0);
const int nsh = 3 * dsh_coefs;          // floats per row of d_shs: 3*M (reference layout) or compact
const int stride = sh_row_stride(p.M);
const int deg = p.sh_degree;
const int ncoef = (deg + 1) * (deg + 1);
if (RAW || shs != nullptr) {
    vis_s[threadIdx.x] = vis;
    __syncthreads();
    if constexpr (RAW) stage_raw_rows<false>(sc.tab, p.M, 3 * ncoef, g0, g_end, vis_s, sh_buf, stride);
    else stage_sh_rows<MT, false>(shs, p.M, 3 * ncoef, g0, g_end, vis_s, sh_buf, stride);   // issue only
}
// every other global load of this thread is issued while the SH rows are still in flight
float x = 0.f, y = 0.f, z = 0.f;
RawShape raw;
float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0;
float4* dg = nullptr;
int grp = 0;                 // RAW: the row's group, its row inside the group and its shape leaves
size_t loc = 0;
RawLeaf lf;
int ci = i;                  // the row's noise counter (LIVE: its compact row)
bool dead = false;           // LIVE: the row is past its group's live count (its radius is 0: not visible)
if constexpr (RAW) {
    if (active) {
        grp = find_group(sc.tab, i);
        loc = (size_t)(i - sc.tab.start[grp]);
        if constexpr (LIVE) { ci = live_row(sc, grp, loc); dead = ci < 0; }
        if (!fz && !dead && (vis || sc.d_scales != nullptr))
            raw_shape(sc.tab, grp, loc, ci, GSR_SEED, GSR_C_SCALE, sc.view, lf, raw);
    }
}
if (vis) {
    if constexpr (RAW) {
        const float* xp = sc.tab.xyz[grp] + 3 * loc;
        x = __ldg(xp); y = __ldg(xp + 1); z = __ldg(xp + 2);
    } else {
        x = __ldg(means3D + 3 * (size_t)i); y = __ldg(means3D + 3 * (size_t)i + 1); z = __ldg(means3D + 3 * (size_t)i + 2);
        load_shape(scales, rots, cov3d, i, raw);
    }
    dg = reinterpret_cast<float4*>(dgeom + 12 * (size_t)(rec_base + i));
    a0 = dg[0]; a1 = dg[1]; a2 = dg[2];
}
if (RAW || shs != nullptr) {
    cp_async_wait_all();
    __syncthreads();
}
if constexpr (RAW) {         // the visible rows' SH coefficients as the forward augmented them (own row)
    if (vis && GSR_C_SHS != 0.0f)
        raw_sh_noise<false>(sh_buf + threadIdx.x * stride, 3 * ncoef, (size_t)ci * 3 * p.M, GSR_SEED,
                            kStreamShs + 2u * sc.view, GSR_C_SHS);
}
float dmean[3] = {0.f, 0.f, 0.f};
float dm2[2] = {0.f, 0.f};
float dop = 0.f;
float dc3o[3] = {0.f, 0.f, 0.f};     // factored SH gradient (dsh_coefs < 0): dL/d(clamped colour), see below
const bool factored = dsh_coefs < 0;
float dsc[3] = {0.f, 0.f, 0.f};
float drot[4] = {0.f, 0.f, 0.f, 0.f};
float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
float dcol[3] = {0.f, 0.f, 0.f};
// composite_bwd (the previous kernel on the stream) has drained its work queue: reset it
if (g_base == 0 && rec_base == 0 && blockIdx.x == 0 && threadIdx.x < GSR_NQUEUE) bwd_queue[threadIdx.x] = 0u;

if (vis) {
    Cam C;
    load_cam(p, C);
    Geo g;
    geo_view(C, x, y, z, g);
    geo_rest(C, p, x, y, z, !RAW && cov3d != nullptr, raw, g);
    // read-and-clear: the accumulators are zero again for the next backward over this `saved`
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    dg[0] = z4; dg[1] = z4; dg[2] = z4;
    const float Wf = (float)p.image_width, Hf = (float)p.image_height;

    // ---- mean2D -------------------------------------------------------------------------
    const float dpx = GSR_PX_GRAD_SCALE * a0.x, dpy = GSR_PX_GRAD_SCALE * a0.y;   // dL/d(pixel mean)
    const float dndcx = dpx * 0.5f * Wf, dndcy = dpy * 0.5f * Hf;
    dm2[0] = dndcx; dm2[1] = dndcy;
    const float pw = g.pw, pw2 = pw * pw;
    const float mul1 = g.hx * pw2, mul2 = g.hy * pw2;
    dmean[0] = (C.F[0] * pw - C.F[3] * mul1) * dndcx + (C.F[1] * pw - C.F[3] * mul2) * dndcy;
    dmean[1] = (C.F[4] * pw - C.F[7] * mul1) * dndcx + (C.F[5] * pw - C.F[7] * mul2) * dndcy;
    dmean[2] = (C.F[8] * pw - C.F[11] * mul1) * dndcx + (C.F[9] * pw - C.F[11] * mul2) * dndcy;

    // ---- opacity, colour ----------------------------------------------------------------
    dop = a1.y;
    const float drgb[3] = {a1.z, a1.w, a2.x};
    const float ddepth = a2.y;

    // ---- conic -> cov2D -----------------------------------------------------------------
    const float ga = -0.5f * a0.z, gb = -a0.w, gc = -0.5f * a1.x;   // dL/d(conic a,b,c)
    const float ca = g.a, cb = g.b, cc = g.c;
    const float di2 = g.det_inv * g.det_inv;
    const float da = (-cc * cc * ga + cb * cc * gb - cb * cb * gc) * di2;
    const float db = (2.f * cb * cc * ga - (ca * cc + cb * cb) * gb + 2.f * ca * cb * gc) * di2;
    const float dc = (-cb * cb * ga + ca * cb * gb - ca * ca * gc) * di2;

    // ---- cov2D -> cov3D (full, unsymmetrised) and -> M ----------------------------------
    float Gs[9];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int k = 0; k < 3; ++k)
            Gs[3 * j + k] = da * g.M0[j] * g.M0[k] + db * g.M0[j] * g.M1[k] + dc * g.M1[j] * g.M1[k];
    float dM0[3], dM1[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        dM0[j] = 2.f * da * g.N0[j] + db * g.N1[j];
        dM1[j] = 2.f * dc * g.N1[j] + db * g.N0[j];
    }
    // M0k = J00*V[4k+0] + J02*V[4k+2] ; M1k = J11*V[4k+1] + J12*V[4k+2]
    float dJ00 = 0.f, dJ02 = 0.f, dJ11 = 0.f, dJ12 = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        dJ00 += dM0[k] * C.V[4 * k + 0];
        dJ02 += dM0[k] * C.V[4 * k + 2];
        dJ11 += dM1[k] * C.V[4 * k + 1];
        dJ12 += dM1[k] * C.V[4 * k + 2];
    }
    const float tz = g.tz, itz = 1.0f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
    const float dcx = -g.fx * itz2 * dJ02;
    const float dcy = -g.fy * itz2 * dJ12;
    float dtz = -g.fx * itz2 * dJ00 - g.fy * itz2 * dJ11 + 2.f * g.fx * g.cx * itz3 * dJ02 +
                2.f * g.fy * g.cy * itz3 * dJ12;
    const float dtx = g.in_x ? dcx : 0.f;
    const float dty = g.in_y ? dcy : 0.f;
    dtz += ddepth;
    dmean[0] += C.V[0] * dtx + C.V[1] * dty + C.V[2] * dtz;
    dmean[1] += C.V[4] * dtx + C.V[5] * dty + C.V[6] * dtz;
    dmean[2] += C.V[8] * dtx + C.V[9] * dty + C.V[10] * dtz;

    if (!RAW && cov3d != nullptr) {
        dcov[0] = Gs[0]; dcov[1] = Gs[1] + Gs[3]; dcov[2] = Gs[2] + Gs[6];
        dcov[3] = Gs[4]; dcov[4] = Gs[5] + Gs[7]; dcov[5] = Gs[8];
    } else {
        // Sigma = L L^T, L = R diag(s): dL = (Gs + Gs^T) L
        float L[9], dLm[9];
#pragma unroll
        for (int r_ = 0; r_ < 3; ++r_)
#pragma unroll
            for (int c_ = 0; c_ < 3; ++c_) L[3 * r_ + c_] = g.R[3 * r_ + c_] * g.s[c_];
#pragma unroll
        for (int r_ = 0; r_ < 3; ++r_)
#pragma unroll
            for (int c_ = 0; c_ < 3; ++c_) {
                float acc = 0.f;
#pragma unroll
                for (int k = 0; k < 3; ++k) acc += (Gs[3 * r_ + k] + Gs[3 * k + r_]) * L[3 * k + c_];
                dLm[3 * r_ + c_] = acc;
            }
        float dR[9];
#pragma unroll
        for (int c_ = 0; c_ < 3; ++c_) {
            dsc[c_] = p.scale_modifier *
                      (dLm[c_] * g.R[c_] + dLm[3 + c_] * g.R[3 + c_] + dLm[6 + c_] * g.R[6 + c_]);
#pragma unroll
            for (int r_ = 0; r_ < 3; ++r_) dR[3 * r_ + c_] = dLm[3 * r_ + c_] * g.s[c_];
        }
        const float4 q = raw.q;
        const float r = q.x, qx = q.y, qy = q.z, qz = q.w;
        drot[0] = 2.f * (-qz * dR[1] + qy * dR[2] + qz * dR[3] - qx * dR[5] - qy * dR[6] + qx * dR[7]);
        drot[1] = 2.f * (qy * dR[1] + qz * dR[2] + qy * dR[3] - 2.f * qx * dR[4] - r * dR[5] +
                         qz * dR[6] + r * dR[7] - 2.f * qx * dR[8]);
        drot[2] = 2.f * (-2.f * qy * dR[0] + qx * dR[1] + r * dR[2] + qx * dR[3] + qz * dR[5] -
                         r * dR[6] + qz * dR[7] - 2.f * qy * dR[8]);
        drot[3] = 2.f * (-2.f * qz * dR[0] - r * dR[1] + qx * dR[2] + r * dR[3] - 2.f * qz * dR[4] +
                         qy * dR[5] + qx * dR[6] + qy * dR[7]);
    }

    // ---- colour -> SH (coefficients live in this thread's shared-memory row) -------------
    if (RAW || shs != nullptr) {
        float vx = x - C.cam[0], vy = y - C.cam[1], vz = z - C.cam[2];
        float dn = sqrtf(vx * vx + vy * vy + vz * vz);
        if (dn == 0.0f) dn = 1.0f;
        const float inv_n = 1.0f / dn;
        const float X = vx / dn, Y = vy / dn, Z = vz / dn;
        float* row = sh_buf + threadIdx.x * stride;
        const int nf = 3 * ncoef;
        float B[16], raw[3];
        sh_basis(deg, X, Y, Z, B);
        sh_color(B, row, nf, raw);
        float dc3[3];
#pragma unroll
        for (int c_ = 0; c_ < 3; ++c_) { dc3[c_] = (raw[c_] < 0.0f) ? 0.0f : drgb[c_]; dc3o[c_] = dc3[c_]; }
        // s_k = sum_c dL/drgb_c * sh[k][c]; then overwrite the row with dL/dsh (float4 chunks)
        float s[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) s[k] = 0.f;
        float4* r4 = reinterpret_cast<float4*>(row);
#pragma unroll
        for (int q = 0; q < 12; ++q) {
            if (4 * q < nf) {
                const float4 v = r4[q];
                const float vv[4] = {v.x, v.y, v.z, v.w};
                float o[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int f = 4 * q + e;
                    o[e] = 0.f;
                    if (f < nf) {
                        s[f / 3] = fmaf(dc3[f % 3], vv[e], s[f / 3]);
                        o[e] = B[f / 3] * dc3[f % 3];
                    }
                }
                if (!factored) r4[q] = make_float4(o[0], o[1], o[2], o[3]);
            }
        }
        if (deg > 0) {
            float gx = -SH_C1 * s[3], gy = -SH_C1 * s[1], gz = SH_C1 * s[2];
            if (deg > 1) {
                gx += SH_C2_0 * Y * s[4] + SH_C2_2 * (-2.f * X) * s[6] + SH_C2_3 * Z * s[7] + SH_C2_4 * 2.f * X * s[8];
                gy += SH_C2_0 * X * s[4] + SH_C2_1 * Z * s[5] + SH_C2_2 * (-2.f * Y) * s[6] + SH_C2_4 * (-2.f * Y) * s[8];
                gz += SH_C2_1 * Y * s[5] + SH_C2_2 * 4.f * Z * s[6] + SH_C2_3 * X * s[7];
                if (deg > 2) {
                    const float xx = X * X, yy = Y * Y, zz = Z * Z;
                    gx += SH_C3_0 * 6.f * X * Y * s[9] + SH_C3_1 * Y * Z * s[10] + SH_C3_2 * (-2.f * X * Y) * s[11] +
                          SH_C3_3 * (-6.f * X * Z) * s[12] + SH_C3_4 * (4.f * zz - 3.f * xx - yy) * s[13] +
                          SH_C3_5 * 2.f * X * Z * s[14] + SH_C3_6 * (3.f * xx - 3.f * yy) * s[15];
                    gy += SH_C3_0 * (3.f * xx - 3.f * yy) * s[9] + SH_C3_1 * X * Z * s[10] +
                          SH_C3_2 * (4.f * zz - xx - 3.f * yy) * s[11] + SH_C3_3 * (-6.f * Y * Z) * s[12] +
                          SH_C3_4 * (-2.f * X * Y) * s[13] + SH_C3_5 * (-2.f * Y * Z) * s[14] +
                          SH_C3_6 * (-6.f * X * Y) * s[15];
                    gz += SH_C3_1 * X * Y * s[10] + SH_C3_2 * 8.f * Y * Z * s[11] +
                          SH_C3_3 * (6.f * zz - 3.f * xx - 3.f * yy) * s[12] + SH_C3_4 * 8.f * X * Z * s[13] +
                          SH_C3_5 * (xx - yy) * s[14];
                }
            }
            // through d = v/|v|
            const float dotg = X * gx + Y * gy + Z * gz;
            dmean[0] += (gx - X * dotg) * inv_n;
            dmean[1] += (gy - Y * dotg) * inv_n;
            dmean[2] += (gz - Z * dotg) * inv_n;
        }
    } else {
        dcol[0] = drgb[0]; dcol[1] = drgb[1]; dcol[2] = drgb[2];
    }
}

if constexpr (RAW) {
    // ---- leaf gradients.  View 0 writes every row (zeros on culled rows); a later view adds into the rows it
    // touched: its visible rows, and every row's _scaling when the augmented scales have an incoming gradient.
    const bool first = sc.view == 0;
    const bool has_ds = sc.d_scales != nullptr && !dead;      // a dead row's scales gradient is zero
    if (active) {
        if (!STATS || d_means2D != nullptr) {
            d_means2D[3 * (size_t)i] = dm2[0]; d_means2D[3 * (size_t)i + 1] = dm2[1]; d_means2D[3 * (size_t)i + 2] = 0.f;
        }
        if constexpr (STATS) {
            // visible = radii > 0 (no row of a group with statistics is frozen: refused on the host)
            const int sv = DYN ? (sc.st.view_dev != nullptr ? __ldg(sc.st.view_dev) : -1) : sc.st.view;
            float* pa = sc.st.accum[grp];
            if (vis && sv == (int)sc.view && pa != nullptr) {
                const int r = __ldg(radii + rec_base + i);
                pa[loc] += gsr_screen_grad_norm(dm2[0], dm2[1]);
                sc.st.denom[grp][loc] += 1.0f;
                float* pm = sc.st.max_radii[grp];
                if (pm != nullptr) pm[loc] = fmaxf(pm[loc], (float)r);
            }
        }
        // this view's contribution to the row's 11 leaf floats; a later view loads all old values before it
        // stores any (the five leaf arrays may alias as far as the compiler knows: load/store pairs would
        // serialise on the load latency)
        float gm[3] = {dmean[0], dmean[1], dmean[2]}, go = 0.0f, gs[3] = {0.f, 0.f, 0.f};
        float4 gq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (vis) {
            const float sig = act_opacity(__ldg(sc.tab.opacity[grp] + loc));
            go = dop * sig * (1.0f - sig);
            gq = quat_normalize_grad(lf.q, lf.nrm, make_float4(drot[0], drot[1], drot[2], drot[3]));
        }
        if (!fz && (vis || has_ds)) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float d = dsc[k] + (has_ds ? __ldg(sc.d_scales + 3 * (size_t)i + k) : 0.0f);
                if (GSR_C_SCALE != 0.0f) d = aug_scale_grad(d, lf.e[k], lf.z[k], GSR_C_SCALE);
                gs[k] = d * lf.e[k];
            }
        }
        float* px = sc.gtab.xyz[grp] + 3 * loc;
        float* po = sc.gtab.opacity[grp] + loc;
        float* ps = sc.gtab.scaling[grp] + 3 * loc;
        float4* pq = reinterpret_cast<float4*>(sc.gtab.rotation[grp]) + loc;
        const bool rows_touched = !fz && (first || vis), scale_touched = !fz && (first || vis || has_ds);
        if (!first) {
            if (rows_touched) {
                const float4 oq = *pq;
                const float ox = px[0], oy = px[1], oz = px[2], oo = *po;
                gm[0] += ox; gm[1] += oy; gm[2] += oz; go += oo;
                gq.x += oq.x; gq.y += oq.y; gq.z += oq.z; gq.w += oq.w;
            }
            if (scale_touched) {
                const float s0 = ps[0], s1 = ps[1], s2 = ps[2];
                gs[0] += s0; gs[1] += s1; gs[2] += s2;
            }
        }
        if (rows_touched) {
            px[0] = gm[0]; px[1] = gm[1]; px[2] = gm[2]; *po = go; *pq = gq;
        }
        if (scale_touched) { ps[0] = gs[0]; ps[1] = gs[1]; ps[2] = gs[2]; }
    }
    // SH: the row holds dL/d(augmented coefficient); times 1 + z c it is the leaf gradient.  Then the rows drain
    // to f_dc / f_rest, half a warp per row (the leaves' rows are not 16-byte aligned).
    const int nf = 3 * ncoef, nrow = 3 * p.M;
    if (vis && GSR_C_SHS != 0.0f)
        raw_sh_noise<true>(sh_buf + threadIdx.x * stride, nf, (size_t)ci * nrow, GSR_SEED, kStreamShs + 2u * sc.view,
                           GSR_C_SHS);
    __syncthreads();
    // Half a warp per row, four rows per thread at a time: a later view loads the old values of all of them
    // before it stores, so twelve loads are in flight instead of one.
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int hl = lane & 15, hsel = lane >> 4;
    const int lim = first ? nrow : nf;                 // view 0 also writes the zeros above the degree
#pragma unroll 1
    for (int it0 = 0; it0 < kBlock / 8; it0 += 4) {
        float* dst[4][3];
        float val[4][3];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int row = (it0 + u) * 8 + w * 2 + hsel;
            const int gi = g0 + row;
            const bool v = gi < g_end && vis_s[row];
            bool on = gi < g_end && (first || v);
            int gg = 0;
            if (on) gg = find_group(sc.tab, gi);
            if constexpr (FROZEN) on = on && !((sc.frozen >> gg) & 1u);
            const size_t ll = on ? (size_t)(gi - sc.tab.start[gg]) : 0;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const int col = hl + 16 * j;
                dst[u][j] = nullptr;
                val[u][j] = 0.0f;
                if (on && col < lim) {
                    dst[u][j] = col < 3 ? sc.gtab.f_dc[gg] + 3 * ll + col : sc.gtab.f_rest[gg] + (size_t)(nrow - 3) * ll + (col - 3);
                    if (v && col < nf) val[u][j] = sh_buf[row * stride + col];
                }
            }
        }
        if (!first) {
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int j = 0; j < 3; ++j)
                    if (dst[u][j]) val[u][j] += *dst[u][j];
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                if (dst[u][j]) *dst[u][j] = val[u][j];
    }
    return;
}

// ---- dense writes (zeros for culled Gaussians).  `accumulate` (bit per output: 1 means3D, 2 opacity,
// 4 sh/colour, 8 scales, 16 rotations, 32 cov3D) adds into the output instead: later views of a multi-view
// backward that share the parameter with an earlier view.
#define GSR_OUT(ptr, val, bit) do { float* p_ = (ptr); *p_ = (accumulate & (bit)) ? *p_ + (val) : (val); } while (0)
if (active) {
    GSR_OUT(d_means3D + 3 * (size_t)i, dmean[0], 1); GSR_OUT(d_means3D + 3 * (size_t)i + 1, dmean[1], 1);
    GSR_OUT(d_means3D + 3 * (size_t)i + 2, dmean[2], 1);
    d_means2D[3 * (size_t)i] = dm2[0]; d_means2D[3 * (size_t)i + 1] = dm2[1]; d_means2D[3 * (size_t)i + 2] = 0.f;
    GSR_OUT(d_opac + i, dop, 2);
    if (cov3d != nullptr) {
#pragma unroll
        for (int k = 0; k < 6; ++k) GSR_OUT(d_cov3d + 6 * (size_t)i + k, dcov[k], 32);
    } else {
        GSR_OUT(d_scales + 3 * (size_t)i, dsc[0], 8); GSR_OUT(d_scales + 3 * (size_t)i + 1, dsc[1], 8);
        GSR_OUT(d_scales + 3 * (size_t)i + 2, dsc[2], 8);
        float4* dr = reinterpret_cast<float4*>(d_rots) + i;
        float4 rv = make_float4(drot[0], drot[1], drot[2], drot[3]);
        if (accumulate & 16) { const float4 o = *dr; rv.x += o.x; rv.y += o.y; rv.z += o.z; rv.w += o.w; }
        *dr = rv;
    }
    if (shs == nullptr) {
        GSR_OUT(d_colors + 3 * (size_t)i, dcol[0], 4); GSR_OUT(d_colors + 3 * (size_t)i + 1, dcol[1], 4);
        GSR_OUT(d_colors + 3 * (size_t)i + 2, dcol[2], 4);
    }
}
if (shs != nullptr && factored) {
    // Factored SH gradient: dL/dsh[k][c] = basis_k(view direction) * dL/d(clamped colour)[c], so the three
    // colour gradients are all another rank needs to rebuild this view's [M, 3] rows (it knows the mean and
    // this view's camera centre): the multi-GPU payload drops from 3*M to 3 floats per Gaussian
    // (b200gsr_sh_grad_expand).  d_shs is a [P, 3] array here.
    if (active) {
        GSR_OUT(d_shs + 3 * (size_t)i, dc3o[0], 4); GSR_OUT(d_shs + 3 * (size_t)i + 1, dc3o[1], 4);
        GSR_OUT(d_shs + 3 * (size_t)i + 2, dc3o[2], 4);
    }
} else if (shs != nullptr) {
    // drain the rows with coalesced stores (zeros for culled rows / inactive degrees)
    __syncthreads();
    const int nf = 3 * ncoef, nchunk = (nf + 3) >> 2;
    if (dsh_coefs != p.M) {
        // compact rows (only the active degree's coefficients, e.g. the NCCL payload at sh_degree 0):
        // the block's rows are one contiguous span of floats, written with coalesced 4-byte stores
        const int rows = min(kBlock, g_end - g0);
        float* base = d_shs + (size_t)g0 * nsh;
        for (int f = threadIdx.x; f < rows * nsh; f += kBlock) {
            const int row = f / nsh, col = f - row * nsh;
            const float val = (vis_s[row] && col < nf) ? sh_buf[row * stride + col] : 0.0f;
            base[f] = (accumulate & 4) ? base[f] + val : val;
        }
    } else if (MT > 0 && ((3 * MT) & 3) == 0) {
        constexpr int q4 = (3 * (MT > 0 ? MT : 4)) / 4;
        float* base = d_shs + (size_t)g0 * 3 * MT;
#pragma unroll
        for (int it = 0; it < q4; ++it) {
            const int u = it * kBlock + threadIdx.x;
            const int row = u / q4, c4 = u - row * q4;
            if (g0 + row < g_end) {
                float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
                if (c4 < nchunk && vis_s[row]) val = *reinterpret_cast<const float4*>(sh_buf + row * stride + 4 * c4);
                if (accumulate & 4) {
                    const float4 o = ldg_f4(base + 4 * u);
                    val.x += o.x; val.y += o.y; val.z += o.z; val.w += o.w;
                }
                stg_na_f4(base + 4 * u, val);
            }
        }
    } else {
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        const int hl = lane & 15, hsel = lane >> 4;
        const bool vec = (nsh & 3) == 0;
        for (int it = 0; it < kBlock / 8; ++it) {
            const int row = it * 8 + w * 2 + hsel;
            if (g0 + row >= g_end) continue;
            float* dst = d_shs + (size_t)(g0 + row) * nsh;
            const bool v = vis_s[row];
            if (vec) {
                for (int q = hl; 4 * q < nsh; q += 16) {
                    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (v && q < nchunk) val = *reinterpret_cast<const float4*>(sh_buf + row * stride + 4 * q);
                    if (accumulate & 4) {
                        const float4 o = ldg_f4(dst + 4 * q);
                        val.x += o.x; val.y += o.y; val.z += o.z; val.w += o.w;
                    }
                    stg_na_f4(dst + 4 * q, val);
                }
            } else {
                for (int col = hl; col < nsh; col += 16) {
                    const float val = (v && col < nf) ? sh_buf[row * stride + col] : 0.0f;
                    dst[col] = (accumulate & 4) ? dst[col] + val : val;
                }
            }
        }
    }
}
