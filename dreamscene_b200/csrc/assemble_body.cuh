// The statements of assemble_kernel and assemble_bwd_frozen_kernel (assemble.cu), included into the body of each.
// In scope: the kernel's parameters, the compile-time BACKWARD and FROZEN, and `frozen` (bit g = group g is frozen;
// a constant 0 in assemble_kernel).  FROZEN: a frozen group's rows are skipped before any load of theirs - no raw
// leaf, noise, packed gradient or leaf gradient is read or written for them.
const int r0 = blockIdx.x * kAsmBlock;
const int i = r0 + threadIdx.x;
if constexpr (FROZEN) {
    // a block whose rows all belong to frozen (or empty) groups returns before any load
    const int last = min(r0 + kAsmBlock, P) - 1;
    bool all = true;
    for (int g = find_group(tab, r0), ge = find_group(tab, last); g <= ge; ++g)
        all = all && (((frozen >> g) & 1u) || tab.start[g + 1] == tab.start[g]);
    if (all) return;
}
// ---- phase A ---------------------------------------------------------------------------
if (i < P) {
    const int g = find_group(tab, i);
    if (!FROZEN || !((frozen >> g) & 1u)) {
        const int l = i - tab.start[g];
        const float sx = tab.scaling[g][3 * (size_t)l], sy = tab.scaling[g][3 * (size_t)l + 1], sz = tab.scaling[g][3 * (size_t)l + 2];
        const float4 q = *reinterpret_cast<const float4*>(tab.rotation[g] + 4 * (size_t)l);
        const float o = tab.opacity[g][l];
        const float e[3] = {act_scale(sx), act_scale(sy), act_scale(sz)};
        const float sig = act_opacity(o);
        const float nrm = quat_norm(q);
        float dsum[3] = {0.f, 0.f, 0.f};
        for (int v = 0; v < B; ++v) {
            float zs[3] = {0.f, 0.f, 0.f};
            if (c_scale != 0.0f) {
                if (z_scales != nullptr) {
                    const float* zr = z_scales + ((size_t)v * P + i) * 3;
                    zs[0] = zr[0]; zs[1] = zr[1]; zs[2] = zr[2];
                } else {
                    const float4 n = normal4(seed, kStreamScales + 2u * (uint32_t)v, (unsigned long long)i);
                    zs[0] = n.x; zs[1] = n.y; zs[2] = n.z;
                }
            }
            float* sv = scales + ((size_t)v * P + i) * 3;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (!BACKWARD) {
                    sv[k] = (c_scale != 0.0f) ? aug_scale(e[k], zs[k], c_scale) : e[k];
                } else {
                    float d = sv[k];
                    if (c_scale != 0.0f) d = aug_scale_grad(d, e[k], zs[k], c_scale);
                    dsum[k] += d;
                }
            }
        }
        if (!BACKWARD) {
            means3D[3 * (size_t)i] = tab.xyz[g][3 * (size_t)l];
            means3D[3 * (size_t)i + 1] = tab.xyz[g][3 * (size_t)l + 1];
            means3D[3 * (size_t)i + 2] = tab.xyz[g][3 * (size_t)l + 2];
            opac[i] = sig;
            *reinterpret_cast<float4*>(rots + 4 * (size_t)i) = quat_normalize(q, nrm);
        } else {
            // incoming gradients live in the packed arrays; outputs are the per-group leaf gradients
            gtab.xyz[g][3 * (size_t)l] = means3D[3 * (size_t)i];
            gtab.xyz[g][3 * (size_t)l + 1] = means3D[3 * (size_t)i + 1];
            gtab.xyz[g][3 * (size_t)l + 2] = means3D[3 * (size_t)i + 2];
            gtab.opacity[g][l] = opac[i] * sig * (1.0f - sig);
#pragma unroll
            for (int k = 0; k < 3; ++k) gtab.scaling[g][3 * (size_t)l + k] = dsum[k] * e[k];
            const float4 gq = *reinterpret_cast<const float4*>(rots + 4 * (size_t)i);
            *reinterpret_cast<float4*>(gtab.rotation[g] + 4 * (size_t)l) = quat_normalize_grad(q, nrm, gq);
        }
    }
}
// ---- phase B: SH rows of the block as a flat span ----------------------------------------
const int rows = min(kAsmBlock, P - r0);
if (rows <= 0) return;
const int row_f = 3 * M;
const size_t base = (size_t)r0 * row_f;          // first float of the block's span in one view's packed array
const size_t view_f = (size_t)P * row_f;         // floats per view
const int total = rows * row_f;
const bool vec = (row_f & 3) == 0;
const int step = vec ? 4 : 1;
for (int f = threadIdx.x * step; f < total; f += kAsmBlock * step) {
    const int row = f / row_f, col = f - row * row_f;       // vec: all 4 elements share the row
    const int gi = r0 + row;
    const int g = find_group(tab, gi);
    if (FROZEN && ((frozen >> g) & 1u)) continue;
    const size_t l = (size_t)(gi - tab.start[g]);
    float raw[4] = {0.f, 0.f, 0.f, 0.f}, dsum[4] = {0.f, 0.f, 0.f, 0.f};
    if (!BACKWARD) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (k >= step) break;
            const int c = col + k;
            raw[k] = (c < 3) ? tab.f_dc[g][3 * l + c] : tab.f_rest[g][(size_t)(row_f - 3) * l + (c - 3)];
        }
    }
    for (int v = 0; v < B; ++v) {
        float z[4] = {0.f, 0.f, 0.f, 0.f};
        const size_t e0 = base + f;                          // element index inside the view
        if (c_shs != 0.0f) {
            if (z_shs != nullptr) {
#pragma unroll
                for (int k = 0; k < 4; ++k) if (k < step) z[k] = z_shs[(size_t)v * view_f + e0 + k];
            } else {
                const float4 n = normal4(seed, kStreamShs + 2u * (uint32_t)v, (unsigned long long)(e0 >> 2));
                if (vec) { z[0] = n.x; z[1] = n.y; z[2] = n.z; z[3] = n.w; }
                else z[0] = (e0 & 3) == 0 ? n.x : (e0 & 3) == 1 ? n.y : (e0 & 3) == 2 ? n.z : n.w;
            }
        }
        float* sv = shs + (size_t)v * view_f + e0;
        if (!BACKWARD) {
            float out[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) out[k] = (c_shs != 0.0f) ? aug(raw[k], z[k], c_shs, 1.0f) : raw[k];
            if (vec) *reinterpret_cast<float4*>(sv) = make_float4(out[0], out[1], out[2], out[3]);
            else sv[0] = out[0];
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (k >= step) break;
                float d = sv[k];
                if (c_shs != 0.0f) d *= (1.0f + z[k] * c_shs);           // d(v + z*(c*v))/dv
                dsum[k] += d;
            }
        }
    }
    if (BACKWARD) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (k >= step) break;
            const int c = col + k;
            if (c < 3) gtab.f_dc[g][3 * l + c] = dsum[k];
            else gtab.f_rest[g][(size_t)(row_f - 3) * l + (c - 3)] = dsum[k];
        }
    }
}
