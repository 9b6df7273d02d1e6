// The select warps of search_topk_kernel (search.cu), as TEXT: this file is #included three times INSIDE the kernel body
// (CRAG_SELECT_SECTION = 1: the tile permutation, 2: the selector state's initialisation, 3: the whole select-warp
// branch), so the kernel compiles from exactly the token stream it had when these lines stood in search.cu -- its
// SASS is byte-identical -- while tests/warp_emu/select_emu_test.cpp includes the same three sections inside a host
// function whose locals carry the same names (keys, thr_key, cnt, pool, k, nq, warp, lane, ...), maps the score-tile
// read (ld_score_row) to a score matrix it supplies and the mbarrier / named-barrier operations to the fiber emulator, and so runs the
// selector of the headline kernel on the CPU: admission, warp-ballot compaction, flushes, pooled floor refreshes,
// rank continuation, the score-all and IVF variants, the drain and the (min, max) reduction.
// Not a header: it has no include guard and declares nothing at namespace scope.
#if CRAG_SELECT_SECTION == 1
  const int perm_groups = perm_mul ? (num_tiles >> perm_shift) : 0;
  auto tile_of = [&](int j) -> int {
    if constexpr (IVF) return j;
    else {
      const int g = j >> perm_shift;
      if (g >= perm_groups) return j;
      return (int((uint64_t(uint32_t(g)) * perm_mul) % uint32_t(perm_groups)) << perm_shift) + (j & ((1 << perm_shift) - 1));
    }
  };
#elif CRAG_SELECT_SECTION == 2
  // selector state: empty lists, thresholds at -inf
  for (int i = threadIdx.x; i < kNQ * L::kKeysPerQuery; i += kSearchThreads) keys[i] = 0ull;
  if (threadIdx.x < kNQ) {
    thr_key[threadIdx.x] = 0ull;
    floor_key[threadIdx.x] = 0ull;
    thr_f[threadIdx.x] = -INFINITY;
    cnt[threadIdx.x] = 0;
    // "search after": rank continuation for k > 128 -- only candidates strictly below the previous pass's last key
    const uint64_t b = (after_keys != nullptr && int(threadIdx.x) < nq) ? after_keys[threadIdx.x] : ~0ull;
    bnd_key[threadIdx.x] = b;
    bnd_f[threadIdx.x] = (b == ~0ull) ? INFINITY : (b == 0ull ? -INFINITY : key_score(b));
  }
#elif CRAG_SELECT_SECTION == 3
    const int quad = warp;      // rows quad * 32 .. quad * 32 + 31 of every score tile
    const int ew = warp;        // select-warp index 0..3 (query ownership for flushes)
    float mn[kNQ], mx[kNQ];
#pragma unroll
    for (int q = 0; q < kNQ; ++q) { mn[q] = INFINITY; mx[q] = -INFINITY; }

    // direct first tile needs room for 128 keys per query and no continuation bound
    const bool direct_first = !IVF && (KLIST + CAP >= 128) && after_keys == nullptr;
    // publish this CTA's best kPoolM rows of query q (call after a flush, by the warp that owns q)
    auto publish = [&](int q) {
      if (pool != nullptr && lane < kPoolM) {
        const uint64_t kk = keys[q * L::kKeysPerQuery + lane];
        if (kk) pool[(size_t(blockIdx.x) * kPoolSlots + lane) * kNQ + q] = kk;
      }
      if (pool != nullptr && lane == kPoolM) {
        // this CTA's own k-th key: it alone holds k rows at or above it, so the MAXIMUM of these over the CTAs is a
        // floor too -- the tight one when scores tie massively (duplicate rows), where a CTA's best keys all sit in
        // one tile and the pooled best keys trail far behind the true k-th key
        const uint64_t kth = keys[q * L::kKeysPerQuery + k - 1];
        if (kth) pool[(size_t(blockIdx.x) * kPoolSlots + kPoolM) * kNQ + q] = kth;
      }
    };
    // raise the thresholds to the pooled floor (all four select warps; see the comment at kPoolM)
    auto raise_to = [&](int q, uint64_t pf) {
      if (q < nq && pf > floor_key[q]) {
        floor_key[q] = pf;
        if (pf > thr_key[q]) {
          thr_key[q] = pf;
          thr_f[q] = key_score(pf);
        }
      }
    };
    auto refresh = [&]() {
      if (pool == nullptr) return;
      if (k <= kPoolSmallK) {
        // lane = query: every warp scans a quarter of the CTAs' best keys, the floor is the minimum of the four
        part_floor[ew * kNQ + lane] = lane_kth_of_pool<4>(pool, int(gridDim.x), ew, lane, 1, (k + 3) / 4);
        named_bar_sync(1, kEpiThreads);
        if (lane < kNQ / 4) {                      // this warp owns queries ew, ew + 4, ...
          const int q = ew + 4 * lane;
          uint64_t pf = part_floor[q];
#pragma unroll
          for (int w2 = 1; w2 < 4; ++w2) pf = part_floor[w2 * kNQ + q] < pf ? part_floor[w2 * kNQ + q] : pf;
          raise_to(q, pf);
        }
        for (int q = ew; q < nq; q += 4) {           // and the largest own-k-th key of any CTA
          const uint64_t mk = pooled_max_kth(pool, int(gridDim.x), q, lane);
          if (lane == 0) raise_to(q, mk);
        }
      } else if (5 * k <= 4 * int(gridDim.x)) {
        // k below the CTA count: the CTAs' best keys suffice; this warp's eight queries are bisected together
        uint64_t pf[8];
        const uint32_t ties = pooled_floor_batch8(pool, int(gridDim.x), ew, nq, k, lane, pf);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int q = ew + 4 * j;
          // the CTAs' own k-th keys are consulted only where scores tie (it costs 5 loads + 2 reductions per query)
          const uint64_t mk = (q < nq && ((ties >> j) & 1u)) ? pooled_max_kth(pool, int(gridDim.x), q, lane) : 0ull;
          if (lane == 0) raise_to(q, mk > pf[j] ? mk : pf[j]);
        }
      } else {
        for (int q = ew; q < nq; q += 4) {
          const uint64_t pf = pooled_kth_key(pool, int(gridDim.x), q, k, lane);
          const uint64_t mk = pooled_max_kth(pool, int(gridDim.x), q, lane);
          if (lane == 0) raise_to(q, mk > pf ? mk : pf);
        }
      }
    };
    // after a flush of query q (lane 0 of the owning warp): threshold = max(local k-th key, pooled floor)
    auto settle = [&](int q) {
      uint64_t t = thr_key[q];
      if (floor_key[q] > t) { t = floor_key[q]; thr_key[q] = t; }
      thr_f[q] = t ? key_score(t) : -INFINITY;
    };
    int acc = 0;
    uint32_t acc_phase = 0;
    int it = 0;
    for (int j = blockIdx.x; j < num_tiles; j += gridDim.x, ++it) {
      const int tile = tile_of(j);
      // after tiles 2, 12, 48 and every 128th: all four warps take the same branch (it is CTA-uniform); the smem
      // thresholds they update are read again only after the next named barrier.  (After two tiles per CTA the pool
      // already holds the best of ~38k rows; what is admitted later is k * ln(rows / 38k) keys per query over ALL
      // CTAs, so further refreshes are for long scans and drifting corpora only.)
      const bool due = k <= kPoolSmallK ? (it == 2 || it == 12 || it == 48 || (it >= 128 && (it & 127) == 0))
                                        : (it == 2 || it == 4 || it == 8 || it == 16 || it == 32 || (it >= 64 && (it & 63) == 0));
      if (due) {
        refresh();
        named_bar_sync(1, kEpiThreads);
      }
      mbar_wait(&bar_tfull[acc], acc_phase);
      uint32_t r[kNQ];
      ld_score_row(score_tiles + acc * (kTileRows * kNQ), quad * 32 + lane, r);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar_tempty[acc]);
      if (++acc == kAccStages) { acc = 0; acc_phase ^= 1; }

      if constexpr (SCORES) {
        const int srow = tile * kTileRows + quad * 32 + lane;
        if (srow < n_rows) {
          if (ivf.best_id != nullptr) {
            const bool first = ivf.base_id == 0;       // the first centroid block starts every row's running best
            float bs = first ? -INFINITY : ivf.best_score[srow];
            int32_t bi = first ? 0 : ivf.best_id[srow];
#pragma unroll
            for (int q = 0; q < kNQ; ++q) {
              const float s = __uint_as_float(r[q]);
              if (q < nq && s > bs) { bs = s; bi = ivf.base_id + q; }   // strict: ties stay with the smaller id
            }
            ivf.best_score[srow] = bs;
            ivf.best_id[srow] = bi;
          } else {
#pragma unroll
            for (int q = 0; q < kNQ; ++q) {
              const float s = __uint_as_float(r[q]);
              mn[q] = fminf(mn[q], s);
              mx[q] = fmaxf(mx[q], s);
              if (q < nq) ivf.out[int64_t(q) * ivf.ld + srow] = s;
            }
          }
        }
        continue;
      }
      int row;
      uint32_t pending = 0;
      if constexpr (!IVF) {
        row = tile * kTileRows + quad * 32 + lane;
        if (row < n_rows) {
#pragma unroll
          for (int q = 0; q < kNQ; ++q) {
            const float s = __uint_as_float(r[q]);
            mn[q] = fminf(mn[q], s);
            mx[q] = fmaxf(mx[q], s);
            // the float test rejects almost everything; survivors must also beat the current k-th KEY, so rows that
            // only tie its score with a larger row id (duplicate-heavy corpora) do not flood the buffer
            if (s >= thr_f[q] && s <= bnd_f[q] && make_key(s, uint32_t(row)) > thr_key[q]) pending |= 1u << q;
          }
          if (nq < kNQ) pending &= (1u << nq) - 1u;
        }
      } else {
        // this tile belongs to ONE coarse list: only the queries probing it see its rows, and a row's score is
        // q . c_list (coarse pass, fp32) + q . residual (this tile's wgmma)
        const int4 item = __ldg(&ivf.work[tile]);
        row = item.x + quad * 32 + lane;
        if (quad * 32 + lane < item.y) {
          const uint32_t probing = __ldg(&ivf.list_mask[item.z]);
          const float* co = ivf.coarse + size_t(item.z) * kNQ;
#pragma unroll
          for (int q = 0; q < kNQ; ++q) {
            if ((probing >> q) & 1u) {
              const float s = __uint_as_float(r[q]) + __ldg(co + q);
              r[q] = __float_as_uint(s);
              mn[q] = fminf(mn[q], s);
              mx[q] = fmaxf(mx[q], s);
              if (s >= thr_f[q] && s <= bnd_f[q] && make_key(s, uint32_t(row)) > thr_key[q]) pending |= 1u << q;
            }
          }
          if (nq < kNQ) pending &= (1u << nq) - 1u;
        }
      }
      // First tile of an unseeded pass: the lists are empty and every row is a candidate.  Skip the reservation
      // protocol (128-way contended atomics, several flush rounds): each row's key goes straight to slot
      // row_in_tile of the query's buffer and one 128-key sort per query builds the list.
      if (direct_first && it == 0) {
#pragma unroll
        for (int q = 0; q < kNQ; ++q)
          keys[q * L::kKeysPerQuery + quad * 32 + lane] =
              ((pending >> q) & 1u) ? make_key(__uint_as_float(r[q]), uint32_t(row)) : 0ull;
        named_bar_sync(1, kEpiThreads);
        for (int q = ew; q < kNQ; q += 4) {
          // exactly 128 keys are live (slots 0..127): sort those, not the whole KLIST + CAP area
          flush_query<KLIST, 128 - KLIST>(keys + q * L::kKeysPerQuery, 128 - KLIST, k, &thr_key[q], lane);
          if (lane == 0) settle(q);
          publish(q);
        }
        named_bar_sync(1, kEpiThreads);
        continue;
      }
      // Candidates are handed to the per-query buffers warp by warp: only the queries that HAVE a candidate in this
      // warp are visited (a set-bit walk over the OR of the lanes' pending masks), one shared-memory atomic reserves
      // the slots of all of a query's candidates in the warp, and the lanes take consecutive slots by ballot rank.
      // (Round 1 walked all 32 queries in every thread with one atomic per candidate; the k = 100 profile showed
      // that per-tile loop, not the sorts or the floor, as the largest share of the select warps' time.)
      const uint32_t lanes_below = (1u << lane) - 1u;
      while (true) {
        bool want_flush = false;
        uint32_t any = __reduce_or_sync(0xffffffffu, pending);
        while (any) {
          const int q = __ffs(any) - 1;
          any &= any - 1u;
          bool mine = (pending >> q) & 1u;
          uint64_t key = 0ull;
          if (mine) {
            key = make_key(__uint_as_float(pick32(r, q)), uint32_t(row));
            if (key >= bnd_key[q]) {             // rank continuation: at or above the previous pass's last key
              mine = false;
              pending &= ~(1u << q);
            }
          }
          const uint32_t m = __ballot_sync(0xffffffffu, mine);
          if (m == 0u) continue;
          const int leader = __ffs(m) - 1;
          int base = 0;
          if (lane == leader) base = atomicAdd(&cnt[q], __popc(m));
          base = __shfl_sync(0xffffffffu, base, leader);
          if (mine) {
            const int slot = base + __popc(m & lanes_below);
            if (slot < CAP) {
              keys[q * L::kKeysPerQuery + KLIST + slot] = key;
              pending &= ~(1u << q);
            }
          }
          if (base + __popc(m) >= CAP) want_flush = true;
        }
        if (!named_bar_or(1, kEpiThreads, want_flush || pending != 0)) break;
        for (int q = ew; q < kNQ; q += 4) {
          const int c = cnt[q];
          if (c >= CAP) {
            flush_query<KLIST, CAP>(keys + q * L::kKeysPerQuery, CAP, k, &thr_key[q], lane);
            if (lane == 0) {
              settle(q);
              cnt[q] = 0;
            }
            publish(q);
          }
        }
        named_bar_sync(1, kEpiThreads);
        for (uint32_t p2 = pending; p2; p2 &= p2 - 1u) {     // what is left and no longer beats the new k-th key: drop
          const int q = __ffs(p2) - 1;
          if (make_key(__uint_as_float(pick32(r, q)), uint32_t(row)) < thr_key[q]) pending &= ~(1u << q);
        }
      }
    }

    // drain candidate buffers, then publish this CTA's lists and (min, max)
    named_bar_sync(1, kEpiThreads);
    if constexpr (!SCORES) {
      for (int q = ew; q < kNQ; q += 4) {
        const int c = min(cnt[q], CAP);
        if (c > kInsertMax) flush_query<KLIST, CAP>(keys + q * L::kKeysPerQuery, c, k, &thr_key[q], lane);
        else if (c > 0) insert_few<KLIST, CAP>(keys + q * L::kKeysPerQuery, c, k, &thr_key[q], lane);
        __syncwarp();
        uint64_t* dst = part_keys + (size_t(blockIdx.x) * kNQ + q) * k;
        for (int j = lane; j < k; j += 32) dst[j] = keys[q * L::kKeysPerQuery + j];
      }
    }
#pragma unroll
    for (int q = 0; q < kNQ; ++q) {
      float a = mn[q], b = mx[q];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
        b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
      }
      if (lane == q) {
        red[(ew * kNQ + q) * 2 + 0] = a;
        red[(ew * kNQ + q) * 2 + 1] = b;
      }
    }
    named_bar_sync(1, kEpiThreads);
    if (ew == 0) {
      float a = red[lane * 2], b = red[lane * 2 + 1];
#pragma unroll
      for (int w = 1; w < 4; ++w) {
        a = fminf(a, red[(w * kNQ + lane) * 2]);
        b = fmaxf(b, red[(w * kNQ + lane) * 2 + 1]);
      }
      part_minmax[(size_t(blockIdx.x) * kNQ + lane) * 2 + 0] = a;
      part_minmax[(size_t(blockIdx.x) * kNQ + lane) * 2 + 1] = b;
    }
#else
#error "define CRAG_SELECT_SECTION to 1, 2 or 3 before including select_warps.inc.cuh"
#endif
#undef CRAG_SELECT_SECTION
