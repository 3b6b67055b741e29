// search_kernel_defs.cuh -- the __global__ kernels of the search family.  No include guard: search_kernels.cuh includes
// this file twice, with SPTAG_B200_BFS false (namespace sptag_b200) and true (namespace sptag_b200::bfs: EnableBfs's
// breadth-first tree seeding compiled in, WarpSearch's BFS flag).  One text for both, and kernels of their own for BFS,
// so that the kernels without it keep their names and their code.
// ------------------------------------------------------------------------------------------
// kernel: persistent warps pull queries from a global counter
// ------------------------------------------------------------------------------------------
// MINB = minimum resident single-warp CTAs per SM the compiler must allow (caps registers): the PQ variant is
// bound by per-step latency, so more resident queries win (80 registers, 24 per SM)
template <int DIM, bool COSINE, int RPL, bool KDT, bool PQ = false, int ELEM = 0, int MINB = 1>
__global__ void __launch_bounds__(32, MINB) search_kernel(const SearchParams p) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x;
    WarpSearch<DIM, COSINE, RPL, PQ, ELEM, true, false, SPTAG_B200_BFS, SPTAG_B200_SKETCH> w(p, lane);
    w.visited = p.vhash ? p.vhash + (size_t)blockIdx.x * (p.vhash_mask + 1ull) : p.visited + (size_t)blockIdx.x * p.visited_words;
    w.vlog = p.vlog ? p.vlog + (size_t)blockIdx.x * p.vlog_entries : nullptr;
    w.tk = p.topk ? p.topk + (size_t)blockIdx.x * p.topk_pad : nullptr;
    w.ng.g = p.ng_spill + (size_t)blockIdx.x * p.ng_spill_entries;
    w.spt.g = p.spt_spill + (size_t)blockIdx.x * p.spt_spill_entries;
    w.setup_warp(smem);

    for (;;) {
        // unsigned: the output offsets below zero-extend it, so nothing about it has to be kept live across the search
        unsigned q = 0;
        if (lane == 0) q = atomicAdd(p.work_counter, 1u);
        q = __shfl_sync(kFull, q, 0);
        // the re-run launch after a hashed-set launch searches the queries on the overflow list that launch left behind
        if (p.rerun) {
            if (q >= p.rerun[0]) break;
            q = p.rerun[1 + q];
        } else if (q >= (unsigned)p.nq) {
            break;
        }

        // ---- WorkSpace::Reset (WorkSpace.h:265-278) ----
        if (w.vlog == nullptr) {
            uint4* v4 = reinterpret_cast<uint4*>(w.visited);
            const size_t n4 = p.visited_words >> 2;
            for (size_t i = lane; i < n4; i += 32) v4[i] = make_uint4(0, 0, 0, 0);
        }
        w.reset_workspace(p.mres_cap);
        // query -> shared memory (+ registers for the static-DIM variants)
        if (PQ && p.pq_adc) {
            // PQQuantizer::QuantizeVector with ADC on (PQQuantizer.h:141-157): table[i][j] = L2(query sub-vector i,
            // codeword j of sub-space i), built by the warp into its slot's arena
            const float* qrot = reinterpret_cast<const float*>(p.queries + (size_t)q * p.query_stride_bytes);
            float* table = p.adc_tables + (size_t)blockIdx.x * p.pq_m * p.pq_ks;
            const int total = p.pq_m * p.pq_ks;
            for (int t = lane; t < total; t += 32) {
                const int i = t / p.pq_ks;
                table[t] = exact_dist_thread<false>(qrot + (size_t)i * p.pq_dsub, p.codebooks + (size_t)t * p.pq_dsub, p.pq_dsub);
            }
            int* qoff = reinterpret_cast<int*>(w.qs);
            for (int i = lane; i < p.pq_m; i += 32) qoff[i] = i * p.pq_ks;
            w.pq_table = table;
        } else if (PQ) {
            // the (already quantized) query: M code bytes -> row offsets of its SDC table rows
            const unsigned char* qc = p.queries + (size_t)q * p.query_stride_bytes;
            int* qoff = reinterpret_cast<int*>(w.qs);
            for (int i = lane; i < p.pq_m; i += 32) qoff[i] = (i * p.pq_ks + (int)qc[i]) * p.pq_ks;
            w.pq_table = p.sdc;
        } else if (ELEM != 0) {
            const unsigned char* qb = p.queries + (size_t)q * p.query_stride_bytes;
            unsigned char* qd = reinterpret_cast<unsigned char*>(w.qs);
            const int qbytes = p.dim * (ELEM == 3 ? 2 : 1);
            for (int i = lane; i < qbytes; i += 32) qd[i] = qb[i];
        } else {
            const float* qg = reinterpret_cast<const float*>(p.queries + (size_t)q * p.query_stride_bytes);
            // static dims that are multiples of 16 never read the shared copy in the BKT flavour (no tails, no
            // KD split test), so those instantiations keep the query in registers only and give the 3 KB back
            // (128-d rows: the fast path reads the query from shared memory with broadcast LDS.128 and holds no slice)
            constexpr bool kRegsOnly = (DIM == 768) && !KDT;
            constexpr bool kFastRows128 = (DIM == 128) && (ELEM == 0) && !PQ;
            if (!kRegsOnly) {
                for (int i = lane; i < p.dim; i += 32) w.qs[i] = qg[i];
                __syncwarp();
            }
            if (DIM > 0 && !kFastRows128) {
#pragma unroll
                for (int c = 0; c < DIM / 16; ++c) w.qr.q[c] = __ldg(qg + 16 * c + (lane & 15));
            }
        }
        if constexpr (SPTAG_B200_SKETCH) {
            signed char* tq = reinterpret_cast<signed char*>(smem + p.off_sketch);
            w.tq = reinterpret_cast<const unsigned*>(tq);
            w.tq_tail = warp_sketch(reinterpret_cast<const float*>(p.queries + (size_t)q * p.query_stride_bytes), p.dim, tq, lane);
            w.nskipped = 0;
        }
        __syncwarp();

        if (KDT)
            w.kdt_search();
        else
            w.bkt_search();

        // log mode and hashed set: leave the bitmap / table clean for the next query of this slot (the table's log never
        // overflows: it holds the load limit plus one row chunk)
        if (w.vlog != nullptr) {
            __syncwarp();
            if (w.vlog_count <= (int)p.vlog_entries) {
                for (int i = lane; i < w.vlog_count; i += 32) w.visited[w.vlog[i]] = 0u;
            } else {  // the log overflowed: clear everything
                uint4* v4 = reinterpret_cast<uint4*>(w.visited);
                const size_t n4 = p.visited_words >> 2;
                for (size_t i = lane; i < n4; i += 32) v4[i] = make_uint4(0, 0, 0, 0);
            }
            __syncwarp();
        }
        // hashed set filled to its limit: the result is incomplete; the re-run launch searches the query again and writes
        // all of its outputs
        if (w.vset_full()) {
            if (lane == 0) p.overflow[1 + atomicAdd(p.overflow, 1u)] = q;
            __syncwarp();
            continue;
        }
        // ---- QueryResultSet::SortResult: the register list is already ascending by (dist, id) ----
        if (w.tk != nullptr) {
            w.res_sort();
            for (int i = lane; i < p.k; i += 32) {
                const int2 e = w.tk[i];
                w.write_result(q, i, e.x, __int_as_float(e.y));
            }
        } else if (lane < p.k) {
            w.write_result(q, lane, w.tk_id, w.tk_d);
        }
        if (p.out_stats != nullptr && lane == 0) {
            int* s = p.out_stats + (size_t)q * kStatsPerQuery;
            s[0] = w.checked;
            s[1] = w.tree_checked;
            s[2] = w.ng.count;
            s[3] = w.spt.count;
            s[4] = w.ndist;
            s[5] = w.nexpand;
            s[6] = w.ntree;
            s[7] = 0;
        }
        if constexpr (SPTAG_B200_SKETCH) {
            if (lane == 0 && w.nskipped) atomicAdd(p.rows_skipped, (unsigned long long)w.nskipped);
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------
// ResultIterator::Next for a batch of open iterators (ResultIterator.cpp:31-55 -> SearchIndexIterativeNext,
// BKTIndex.cpp:659-675).  Every query owns persistent arenas in HBM -- visited bitmap, NGQueue, SPTQueue (the
// reference's rented WorkSpace) -- indexed by query, not by slot; the shared-memory queue heads are restored from and
// flushed to those arenas around each call, and the rest of its state is an IterState.
// p.k = the batch the caller asked for; the effective batch of a query is capped by the result count of its previous
// call (QueryResult::SetResultNum(resultCount), ResultIterator.cpp:36-41, :52).
// A query on a hash table that reaches the table's limit suspends (bkt_search_iterative): it saves what the call has
// built so far, writes no outputs and joins iv.suspended; the host grows its table and launches the kernel again over
// that list (iv.list), where the query continues from the saved state.  The visited set has exact set semantics in
// both forms, so the results do not depend on where, or how often, a query was suspended.
// ------------------------------------------------------------------------------------------
template <bool COSINE, int RPL, int ELEM>
__global__ void __launch_bounds__(32, 12) iterate_kernel(const SearchParams p, int* __restrict__ state,
                                                         int* __restrict__ out_counts,
                                                         unsigned char* __restrict__ out_relaxed, const IterVisited iv) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x;
    IterState* const states = reinterpret_cast<IterState*>(state);
    WarpSearch<0, COSINE, RPL, false, ELEM, false, true, SPTAG_B200_BFS> w(p, lane);
    w.vlog = nullptr;  // the bitmap belongs to the iterator and is never cleared between calls
    w.setup_warp(smem);

    for (;;) {
        const int q = next_iter_query(p, iv, lane);
        if (q < 0) break;
        IterState& st = states[q];
        bind_iter_visited(w, p, iv, q, st.vbits);
        w.ng.g = p.ng_spill + (size_t)q * p.ng_spill_entries;
        w.spt.g = p.spt_spill + (size_t)q * p.spt_spill_entries;
        w.tk = p.topk + (size_t)q * p.topk_pad;
        w.ng.count = st.ng_count;
        w.spt.count = st.spt_count;
        w.ng.tail_idx = w.spt.tail_idx = -1;
        const int resumed = st.resume;
        int at = resumed ? resumed : (st.first != 0 ? kIterFirst : kIterStep);
        int relaxed = st.relaxed;
        const int slots = st.slots;
        const int batch = (slots < 0) ? p.k : min(p.k, slots);
        w.restore_queue_heads();
        w.ndist = w.nexpand = w.ntree = 0;
        w.tree_checked = w.no_better = 0;
        w.vlog_count = st.vfill;
        float* saved = iv.resume ? iv.resume + (size_t)q * kIterResumeWords : nullptr;
        int count = 0, limit = 0;
        if (resumed) {  // the call this query suspended in: m_Results, resultCount, checked and the SearchTrees limit
            w.mres.load(saved, lane);
            const int* si = reinterpret_cast<const int*>(saved + 32 * RPL);
            count = si[0];
            w.checked = si[1];
            limit = si[2];
        } else {
            // WorkSpace::ResetResult(m_iMaxCheck, batch) (WorkSpace.h:280-286)
            w.mres.reset(max(p.max_check / 16, batch), lane);
            w.checked = 0;
        }
        w.tk_count = count;
        w.load_query_bytes(q);
        __syncwarp();

        w.bkt_search_iterative(at, batch, relaxed, count, limit, iv.margin);

        __syncwarp();
        if (at != kIterDone) {  // suspended: keep the call's state, flush the queues, no outputs yet
            w.mres.save(saved, lane);
            if (lane == 0) {
                int* si = reinterpret_cast<int*>(saved + 32 * RPL);
                si[0] = count;
                si[1] = w.checked;
                si[2] = limit;
            }
            w.flush_queue_heads();
            if (lane == 0) {
                st.ng_count = w.ng.count;
                st.spt_count = w.spt.count;
                st.relaxed = relaxed;
                st.vfill = w.vlog_count;
                st.resume = at;
            }
            suspend_iter_query(iv, q, at == kIterStep ? 1 : 2, lane);
            __syncwarp();
            continue;
        }
        // QueryResultSet::SortResult over the `count` returned entries; the rest of the caller's row is (-1, MaxDist)
        w.res_sort();
        for (int i = lane; i < p.k; i += 32) {
            const int2 e = (i < count) ? w.tk[i] : make_pair(-1, SPTAG_B200_MAXDIST);
            w.write_result(q, i, e.x, __int_as_float(e.y));
        }
        // flush the queue heads and the scalars
        w.flush_queue_heads();
        if (lane == 0) {
            st.ng_count = w.ng.count;
            st.spt_count = w.spt.count;
            st.first = 0;
            st.relaxed = relaxed;
            st.slots = count;  // m_queryResult->SetResultNum(resultCount)
            st.vfill = w.vlog_count;
            st.resume = 0;
            out_counts[q] = count;
            out_relaxed[q] = (unsigned char)relaxed;
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------
// BKT::Index<T>::SearchIndexIterativeFromNeareast, FIRST call (BKTIndex.cpp:543-573), for a batch of freshly opened
// iterators -- the head-index call of SPANN's iterative search (SPANNIndex.cpp:273): a full Search for the p.k nearest on
// the query's own work-space arenas, nodeCheckStatus.clear(), then every result re-seeds NGQueue from its graph row.
// Later calls are iterate_kernel with batch = k (the host resets the result-slot cap: the caller's QueryResult keeps
// its size there).
// The search is not resumable mid-way: a query whose table reaches its limit joins iv.suspended and the host runs its
// call again from the start on a larger, empty table (exact: the iterator was freshly opened).  The host sizes the
// tables so that the seeding (at most k x (degree + 1) inserts) stays below the limit.
// ------------------------------------------------------------------------------------------
template <bool COSINE, int RPL, int ELEM>
__global__ void __launch_bounds__(32, 12) nearest_first_kernel(const SearchParams p, int* __restrict__ state,
                                                               const IterVisited iv) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x;
    IterState* const states = reinterpret_cast<IterState*>(state);
    WarpSearch<0, COSINE, RPL, false, ELEM, false, true, SPTAG_B200_BFS> w(p, lane);
    w.ring = smem;
    w.cand_id = reinterpret_cast<int*>(smem + p.off_cand);
    w.cand_dist = reinterpret_cast<float*>(smem + p.off_cand + 128);
    w.bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
    w.qs = reinterpret_cast<float*>(smem + p.off_query);
    w.vlog = nullptr;
    w.ng.s = reinterpret_cast<int2*>(smem + p.off_ng);
    w.ng.H = p.h_ng;
    w.ng.length = p.ng_length;
    w.ng.lastlevel = p.ng_lastlevel;
    w.spt.s = reinterpret_cast<int2*>(smem + p.off_spt);
    w.spt.H = p.h_spt;
    w.spt.length = p.spt_length;
    w.spt.lastlevel = p.spt_lastlevel;
    w.phase_bits = 0;
    if (lane == 0) {
        for (int s = 0; s < p.stages; ++s) mbar_init(&w.bars[s], 1);
        mbar_fence_init();
        w.ng.s[0] = make_pair(-1, SPTAG_B200_MAXDIST);
        w.spt.s[0] = make_pair(-1, SPTAG_B200_MAXDIST);
    }
    __syncwarp();

    for (;;) {
        const int q = next_iter_query(p, iv, lane);
        if (q < 0) break;
        IterState& st = states[q];
        bind_iter_visited(w, p, iv, q, st.vbits);  // empty: zeroed when the iterator was opened or the table was grown
        w.ng.g = p.ng_spill + (size_t)q * p.ng_spill_entries;
        w.spt.g = p.spt_spill + (size_t)q * p.spt_spill_entries;
        w.tk = (p.k > 32) ? p.topk + (size_t)q * p.topk_pad : nullptr;
        // the rented WorkSpace after Reset(MaxCheck, k) + ResetResult(MaxCheck, k)
        w.vlog_count = 0;
        w.ng.count = 0;
        w.spt.count = 0;
        w.ng.tail_idx = w.spt.tail_idx = -1;
        w.mres.reset(max(p.max_check / 16, p.k), lane);
        w.tk_d = SPTAG_B200_MAXDIST;
        w.tk_id = -1;
        w.worst_d = SPTAG_B200_MAXDIST;
        w.worst_id = -1;
        if (w.tk != nullptr) w.res_reset();
        w.checked = w.ndist = w.nexpand = w.ntree = 0;
        w.tree_checked = w.no_better = 0;
        {
            const unsigned char* qb = p.queries + (size_t)q * p.query_stride_bytes;
            unsigned char* qd = reinterpret_cast<unsigned char*>(w.qs);
            const int qbytes = p.dim * (ELEM == 0 ? 4 : (ELEM == 3 ? 2 : 1));
            for (int i = lane; i < qbytes; i += 32) qd[i] = qb[i];
        }
        __syncwarp();

        w.bkt_search();  // SearchIndex(query, workspace, p_searchDeleted, searchDuplicated = true)

        __syncwarp();
        if (w.vset_full()) {  // the table filled: run the whole call again on a larger one
            suspend_iter_query(iv, q, 0, lane);
            __syncwarp();
            continue;
        }
        if (w.tk != nullptr) w.res_sort();
        // p_space->nodeCheckStatus.clear(): other nodes may be traversed again after the top k were found
        {
            uint4* v4 = reinterpret_cast<uint4*>(w.visited);
            const size_t n4 = w.qmask ? (w.qmask + 1u) >> 2 : p.visited_words >> 2;
            for (size_t i = lane; i < n4; i += 32) v4[i] = make_uint4(0, 0, 0, 0);
        }
        w.vlog_count = 0;
        __syncwarp();
        for (int i = 0; i < p.k; ++i) {
            int rid;
            float rd;
            if (w.tk != nullptr) {
                const int2 e = w.tk[i];
                rid = e.x;
                rd = __int_as_float(e.y);
            } else {
                rid = __shfl_sync(kFull, w.tk_id, i);
                rd = __shfl_sync(kFull, w.tk_d, i);
            }
            if (lane == 0) {
                p.out_ids[(size_t)q * p.k + i] = (rid >= 0) ? rid + p.id_offset : rid;
                p.out_dists[(size_t)q * p.k + i] = rd;
            }
            if (rid < 0) continue;
            w.seed_from_result(rid);
        }
        // flush the queue heads and the scalars
        __syncwarp();
        for (int i = 1 + lane; i <= min(w.ng.count, w.ng.H); i += 32) w.ng.g[i] = w.ng.s[i];
        for (int i = 1 + lane; i <= min(w.spt.count, w.spt.H); i += 32) w.spt.g[i] = w.spt.s[i];
        if (lane == 0) {
            st.ng_count = w.ng.count;
            st.spt_count = w.spt.count;
            st.first = 0;
            st.slots = -1;
            st.vfill = w.vlog_count;
        }
        __syncwarp();
    }
}
