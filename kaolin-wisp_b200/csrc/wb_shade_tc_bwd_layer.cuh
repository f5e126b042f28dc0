// wb_shade_tc_bwd_layer.cuh -- body of the backward layer walk of wb_mlp_bwd_tc_kernel (wb_shade_tc.cu), included twice there: into
// the run-time loop of TcShapeRt (TC_END_LAYERS = break) and into the unrolled walk of a TcShape (TC_END_LAYERS = return; it only
// ends the walk at layer 0, the last one).  One text for both keeps the run-time kernels' code exactly what it is without a TcShape.
// In scope: the kernel's per-tile state, the layer index l (int, or TcInt<l> for a TcShape) and the shape S.
            tc_publish(c);
            const int I = m.I[l], O = m.O[l];
            const auto Kp = S::Kp(m, l);
            const int Np = S::Np(m, l);
            const uint32_t xb = tc_smem_u32(c.sub + m.tile_off[l]);
            // weight grad acc_l^T[out, in] += dY_l^T . X_l and, from the constant-one slab, acc_l^T[out, I] += dY_l^T . 1, one round per
            // block of 64 outputs; the data grad dX_l = dY_l . W_l joins the round of the last block
            const bool wg = m.acc_l[l] >= 0, bg = m.src_b[l] >= 0, dg = l > 0 || emit;
            float* al = acc + m.acc_l[l];
            const uint64_t xw = tc_desc(xb, 128, TC_SLAB), xone = tc_desc(xb + (uint32_t)(Kp / 8) * TC_SLAB, 128, TC_SLAB);
            const uint64_t dyd = tc_desc(dyb, TC_SLAB, 128), wd = tc_desc(wb + m.w_off[l], 128, Np * 16);
            auto rounds = [&](auto d16, auto&& depi) {
                const int nmb = wg ? (Np + 63) / 64 : 1;
                for (int b = 0; b < nmb; ++b) {
                    const int mb = 64 * b;
                    tc_bwd_round_n<decltype(d16)::value>(Kp, c, wg, bg, dg && b == nmb - 1, tc_desc(dyb + (uint32_t)(mb / 8) * TC_SLAB, 128, TC_SLAB),
                                                         xw, xone, dyd, wd, Np / 16,
                        [&](auto& d) {
                            constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                            for (int i = 0; i < NR; ++i) {
                                const int o = mb + tc_frag_row(c.wl, i), k = tc_frag_col(c.wl, i);
                                if (o < O && k < I) al[o * (I + 1) + k] += d[i];
                            }
                        },
                        [&](auto& d) {
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const int o = mb + tc_frag_row(c.wl, i);
                                if (o < O && tc_frag_col(c.wl, i) == 0) al[o * (I + 1) + I] += d[i];
                            }
                        },
                        depi);
                }
            };
            if (!dg) {
                if (wg) rounds(std::false_type(), [](auto&) {});
                TC_END_LAYERS;
            }
            if (l == S::nl_d(m)) {
                // first colour layer: inputs [df[1:dout], embed(ray_d)]; only the first dout-1 <= 15 carry gradient (nerf.py:259)
                rounds(std::true_type(), [&](auto& d) { TC_FRAG_TO_SCRATCH(c, d, 16); });
                tc_sync(c);
                const float* v = c.scr + c.r * TC_SCR_LD;
                const int dout = m.O[S::nl_d(m) - 1];
                float gdf[16];
                gdf[0] = (df[0] > 0.0f) ? go.w * scale : 0.0f;   // relu' of density (nerf.py:263)
#pragma unroll
                for (int j = 1; j < 16; ++j) gdf[j] = (j < dout) ? v[j - 1] : 0.0f;
                if (c.h == 0) tile_store8(dyt, c.r, 0, gdf); else tile_store8(dyt, c.r, 1, gdf + 8);
                for (int sl = 2 + c.h; sl < S::Np(m, tc_step<-1>(l)) / 8; sl += 2) tile_store8(dyt, c.r, sl, z8);
            } else if (l == 0 && FUSE) {
                // dL/d(grid features) -> hash table: column half h holds features [16h, 16h+16) = LODs 8h .. 8h+7; a warp = 32
                // consecutive samples of one half
                rounds(std::false_type(), [&](auto& d) { TC_FRAG_TO_SCRATCH(c, d, 32); });
                tc_sync(c);
                const float* v = c.scr + c.r * TC_SCR_LD + c.h * 16;
                const float3 p = wb_ray_point(in.origins, in.dirs, ray, __ldg(in.rec_t + s));
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int lv = c.h * 8 + q;
                    if (lv < G.planes) tc_scatter_level_f2(g, lv, p, valid, v[2 * q], v[2 * q + 1], inv_scale, lane, gtable);
                }
            } else if (l == 0) {
                // dL/d(grid features) -> fp16 planes [plane][S][width] (still loss-scaled), straight from the fragments
                const int W = G.width, nfe = G.planes * W;
                const int64_t srow0 = tile * TC_ROWS;
                rounds(std::false_type(), [&](auto& d) {
                    constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                    for (int i = 0; i < NR; i += 2) {
                        const int64_t sr = srow0 + tc_frag_row(c.wl, i);
                        const int fe = tc_frag_col(c.wl, i);
                        if (sr >= s_end || fe >= nfe) continue;
                        if (W == 2) reinterpret_cast<__half2*>(G.dfeat)[(int64_t)(fe >> 1) * in.S + sr] = __floats2half2_rn(d[i], d[i + 1]);
                        else {
                            G.dfeat[((int64_t)(fe / W) * in.S + sr) * W + (fe % W)] = __float2half_rn(d[i]);
                            if (fe + 1 < nfe) G.dfeat[((int64_t)((fe + 1) / W) * in.S + sr) * W + ((fe + 1) % W)] = __float2half_rn(d[i + 1]);
                        }
                    }
                });
            } else {
                // hidden layer input: apply relu' from the retained activation tile, write the next dY (Np[l-1] == Kp[l])
                const uint8_t* xt = c.sub + m.tile_off[l];
                rounds(std::false_type(), [&](auto& d) {
                    constexpr int NR = sizeof(d) / sizeof(float);
                    const __half2 z2 = __float2half2_rn(0.0f);
#pragma unroll
                    for (int i = 0; i < NR; i += 2) {
                        const int row = tc_frag_row(c.wl, i), col = tc_frag_col(c.wl, i);
                        const int off = (col >> 3) * TC_SLAB + row * 16 + (col & 7) * 2;
                        // relu'(x) as a 16-bit lane mask of the retained fp16 activation (>= 0 by construction)
                        const uint32_t a = *reinterpret_cast<const uint32_t*>(xt + off);
                        *reinterpret_cast<uint32_t*>(dyt + off) = tc_pack2(d[i], d[i + 1]) & __hgt2_mask(*reinterpret_cast<const __half2*>(&a), z2);
                    }
                });
            }
