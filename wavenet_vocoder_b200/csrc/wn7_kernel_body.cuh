// wn7_kernel_body.cuh — the body of both engine-7 kernels (wn7_kernel.cuh: wn7_kernel and wn7_stream_kernel),
// included inside each __global__ with BT, SELF, STREAM, pl and pp in scope.  A textual include, not a shared
// __forceinline__ function: routing the whole-utterance kernels through such a function changed their SASS
// (same registers, different schedule), and they are meant to compile exactly as without streams.
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Engine<BT, SELF, STREAM> eng(pl, pp, smem_raw);
    const int npollw = SELF ? WN7_NSP : pl.npw;
    const int tid = eng.tid, p = blockIdx.x, warp = eng.warp, NT = pl.nthreads;     // logical indices (see Engine)
    const int nslots = pl.nres + pl.nring;
    const int L = pl.L, RA4 = 4 * pl.qA;
    if (tid == 0) {
        for (int i = 0; i < nslots; ++i) mbar_init(&eng.bar_full_()[i], 1);
        for (int i = 0; i < pl.nring; ++i) mbar_init(&eng.bar_empty_()[i], WN7_NCW);
        for (int i = 0; i < 2; ++i) {
            mbar_init(&eng.bar_cfull_()[i], 1);
            mbar_init(&eng.bar_cempty_()[i], 1);
            mbar_init(&eng.bar_in_()[i], npollw);
            mbar_init(&eng.bar_free_()[i], WN7_NCW);
        }
        mbar_init(eng.bar_pre_(), 1);
        mbar_init(eng.bar_x0_(), npollw);
        mbar_init(eng.bar_ps_(), npollw);
        mbar_init(eng.bar_dstep_(), WN7_NCW);
        mbar_init(&eng.bar_crit_()[0], WN7_NCW);
        mbar_init(&eng.bar_crit_()[1], WN7_NCW);
        *eng.s_abort_() = 0;
        *eng.s_skipcnt_() = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // pass table
    {
        const int nw = pl.npass * (int)(sizeof(Wn7Pass) / 4);
        const int* src = reinterpret_cast<const int*>(pp.passes);
        int* dst = reinterpret_cast<int*>(eng.passes_());
        for (int i = tid; i < nw; i += NT) dst[i] = src[i];
    }
    // zero the history (== the reference's zero-initialised queue, conv.py:35-36) and the scratch buffers; a continued
    // stream loads the history its previous launch stored instead (rings in global memory ARE the state buffer)
    if (pl.ring_in_smem) {
        const size_t n = (size_t)pl.ring_pos_total * RA4 * BT;
        const float* src = nullptr;
        if constexpr (STREAM) {
            if (pp.state_load) src = pp.state + (size_t)p * n;
        }
        for (size_t i = tid; i < n; i += NT) eng.ring_()[i] = src ? src[i] : 0.f;
    }
    for (int i = tid; i < 2 * pl.xin_vals * BT; i += NT) eng.xin_()[i] = 0.f;
    for (int i = tid; i < pl.ms * BT; i += NT) eng.skipacc_()[i] = 0.f;
    for (int i = tid; i < 2 * pl.mx * BT; i += NT) eng.xown_()[i] = 0.f;
    for (int i = tid; i < pl.O * BT + 2; i += NT) eng.hs_()[i] = 0.f;
    for (int i = tid; i < pl.L * (pl.kw - 1); i += NT) {
        eng.ringtab_()[i * 3] = pp.ringtab[i * 2];           // offset of the ring (in positions)
        eng.ringtab_()[i * 3 + 1] = pp.ringtab[i * 2 + 1];   // delay D
        eng.ringtab_()[i * 3 + 2] = STREAM ? (int)(pp.t_base % (unsigned)pp.ringtab[i * 2 + 1]) : 0;   // (absolute t) mod D
    }
    // biases of the rows this block owns
    {
        const float* src = pp.bpack + (size_t)p * pl.cta_b_floats;
        for (int i = tid; i < pl.cta_b_floats; i += NT) eng.bias_()[i] = src[i];
    }
    // first 1x1 conv: [w (scalar input) | b]
    for (int k = tid; k < pl.R; k += NT) {
        eng.x0w_()[k] = (pl.input_kind == 0) ? pp.first_w[k] : 0.f;
        eng.x0w_()[pl.R + k] = pp.first_b[k];
    }
    {
        // static part of the pre-activation: (folded) conv bias + global-conditioning projection
        // (modules.py:148-152 recomputes Wg.g every step although g is constant; fold it once)
        const float* bsrc = pp.bpack + (size_t)p * pl.cta_b_floats + pl.bo_zb;
        const int n = L * RA4 * BT;
        for (int i = tid; i < n; i += NT) {
            const int b = i % BT, rr = (i / BT) % RA4, l = i / (BT * RA4);
            float v = 0.f;
            if ((rr >> 1) < eng.ny) {
                v = bsrc[l * 2 * pl.my + rr];
                if (pp.gbias != nullptr && b < pp.B) {
                    const int grow = (rr & 1) ? pl.G2 + eng.y0 + (rr >> 1) : eng.y0 + (rr >> 1);
                    v += pp.gbias[((size_t)b * L + l) * pl.G + grow];
                }
            }
            eng.sb_()[i] = v;
        }
    }
    // feedback for step 0 (wavenet.py:281-301)
    if (tid < BT) {
        const int b = tid;
        float v = 0.f;
        int idx = -1;
        if (b < pp.B) {
            if (pl.input_kind == 0) {
                if (pp.T_test > 0) v = pp.test_scalar[(size_t)b * pp.T_test];
                else if (pp.initial) v = pp.initial[b];
            } else {
                if (pp.T_test > 0) idx = pp.test_index ? pp.test_index[(size_t)b * pp.T_test] : -1;
                else if (pp.initial_dense) idx = -1;
                else if (pp.initial_rows) idx = pp.initial_rows[b];
                else idx = pp.initial_index;
            }
        } else if (pl.input_kind != 0) idx = 0;
        if constexpr (STREAM) {
            if (pp.state_load) {                 // the feedback the previous launch left
                const float* fb = pp.state + (size_t)pl.P * wn7_state_ring_floats(pl);
                v = fb[b];
                idx = __float_as_int(fb[BT + b]);
            }
        }
        eng.s_in_()[b] = v;
        eng.s_idx_()[b] = idx;
    }
    if (pl.input_kind != 0) {
        const float* dsrc = nullptr;
        size_t stride = 0;
        if (pp.T_test > 0 && pp.test_dense != nullptr) { dsrc = pp.test_dense; stride = (size_t)pp.T_test * pl.O; }
        else if (pp.T_test == 0 && pp.initial_dense != nullptr) { dsrc = pp.initial_dense; stride = (size_t)pl.O; }
        const float* fb = nullptr;
        if constexpr (STREAM) {
            if (pp.state_load) fb = pp.state + (size_t)pl.P * wn7_state_ring_floats(pl) + 2 * BT;
        }
        for (int i = tid; i < BT * pl.O; i += NT) {
            const int b = i / pl.O, o = i % pl.O;
            eng.s_dense_()[i] = fb ? fb[i] : ((dsrc && b < pp.B) ? dsrc[(size_t)b * stride + o] : 0.f);
        }
    }
    if (warp < npollw) {
        for (int b = warp; b < BT; b += npollw) eng.fetch_noise(0, b);
    }
    __syncthreads();

    if (warp < pl.npw) eng.poll_loop();
    else if (warp < wn7_warp_hk(pl)) eng.comp_loop();
    else if (warp == wn7_warp_hk(pl)) eng.hk_loop();
    else if (warp == wn7_warp_tma(pl)) eng.tma_loop();
    else if (pl.C > 0) eng.cond_loop();
    if constexpr (STREAM) {
        __syncthreads();                      // every role loop is past its last step: rings and feedback are final
        wn7_store_state<BT>(pl, pp, smem_raw);
    }
