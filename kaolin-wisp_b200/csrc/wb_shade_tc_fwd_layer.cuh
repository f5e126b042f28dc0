// wb_shade_tc_fwd_layer.cuh -- body of the forward layer walk of tc_decoders (wb_shade_tc.cu), included twice there: into the run-time
// loop of TcShapeRt (TC_NEXT_LAYER = continue) and into the unrolled walk of a TcShape (TC_NEXT_LAYER = return).  One text for both
// keeps the run-time kernels' code exactly what it is without a TcShape; wrapping their loop body in a lambda changes their schedule.
// In scope: m, c, in, ray, df, c3, nl, the layer index l (int, or TcInt<l> for a TcShape) and the shape S.
        const bool last_d = (l == S::nl_d(m) - 1), last_c = (l == nl - 1);
        tc_publish(c);
        if (!last_d && !last_c) {
            // hidden layer: relu(acc) -> next input tile (F2FP.RELU), straight from the fragments; Np[l] == Kp[l+1], padded outputs
            // are relu(0 + 0) = 0
            uint8_t* tn = c.sub + m.tile_off[l + 1];
            tc_fwd_layer<NMAX, S>(m, c, l, S::Np(m, l), [&](auto& d) {
                constexpr int NR = sizeof(d) / sizeof(float);
#pragma unroll
                for (int i = 0; i < NR; i += 2) {
                    const int row = tc_frag_row(c.wl, i), col = tc_frag_col(c.wl, i);
                    *reinterpret_cast<uint32_t*>(tn + (col >> 3) * TC_SLAB + row * 16 + (col & 7) * 2) = tc_pack2_relu(d[i], d[i + 1]);
                }
            });
            TC_NEXT_LAYER;
        }
        tc_fwd_layer<NMAX, S>(m, c, l, 16, [&](auto& d) { TC_FRAG_TO_SCRATCH(c, d, 16); });      // both heads are <= 16 wide
        tc_sync(c);
        const float* srow = c.scr + c.r * TC_SCR_LD;
        if (last_d) {
#pragma unroll
            for (int j = 0; j < 16; ++j) df[j] = srow[j];
            // colour input = [df[1:], embed(ray_d)], zero padded (nerf.py:248-259): the per-ray row already holds the
            // embedding and the zero padding, only the first dout-1 (<= 15) features are per-sample.  16-byte chunk ch of the
            // row is written by column half ch & 1.
            uint8_t* tcol = c.sub + m.tile_off[l + 1];
            const int nd = m.O[l] - 1, nch = S::Kp(m, tc_step<1>(l)) / 8;
            const uint4* re = in.ray_embed + ray * nch;
            uint4 q = __ldg(re + c.h);
            __half* hq = reinterpret_cast<__half*>(&q);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                // feature 8*h + j <- df[8*h + j + 1]; select without dynamic register indexing
                const float dv = c.h == 0 ? df[(j + 1) & 15] : df[(j + 9) & 15];
                if (8 * c.h + j < nd) hq[j] = __float2half_rn(dv);
            }
            *reinterpret_cast<uint4*>(tcol + c.h * TC_SLAB + c.r * 16) = q;
            for (int ch = 2 + c.h; ch < nch; ch += 2) *reinterpret_cast<uint4*>(tcol + ch * TC_SLAB + c.r * 16) = __ldg(re + ch);
        } else {
            c3[0] = srow[0]; c3[1] = srow[1]; c3[2] = srow[2];
        }
