// spgemm_stream.cuh -- masked SpGEMM, the chunked classes:  T<M> = A (+).(x) B  where products are kept only on M's pattern.
//
// The triangle kernel C<L> = L (+.pair) L of BASELINE.json configs[3] makes 8e9 products for 1e7 outputs: 96 % of the
// products miss the mask.  The kernel is therefore built around the MISS path:
//
//   * membership filter: a BITMAP of the mask row's columns in shared memory (exact, bit j, when ncols fits; a one-hash
//     Bloom filter otherwise) -- one LDS and a bit test per product instead of a hash probe loop;
//   * B rows are streamed by whole warps with coalesced 128-bit loads of four column ids per lane (one A entry per
//     warp at a time; B rows longer than LONG_ROW positions are cut into 128-position blocks dealt to all the warps);
//   * the survivors (true hits, ~5 % of the products, + filter false positives) are compacted with ballots into a
//     per-warp queue and resolved 32 at a time by all lanes: a shared-memory hash of the mask row (short mask rows) or a
//     dense column -> position map in HBM (hub mask rows) gives the output position in one probe, then the product is
//     combined into a shared-memory accumulator (short mask rows) or straight into HBM;
//   * CTAs are persistent and take blocks of CONSECUTIVE chunks (a chunk = row i + a flop-bounded slice of A(i,:)), so
//     the filter of a hub row is built once and reused by all its chunks; rows are changed by clearing exactly the
//     bits that were set.
//
// Algorithmic bytes (SURVEY.md 8d): flops x (4 + b_B) for the streamed B entries -- they come from the L2 when B fits
// (scale 20: 63 MB of column ids), which is what the coalesced 128-bit loads are for.
#pragma once

struct StreamArgs {
    GemmArgs g;
    const int32_t *chunk_row; const uint32_t *chunk_idx; const uint32_t *chunk_cnt; int64_t nchunks;
    void *t_words;                  // nnz(M) accumulator words (pre-set to accum_init)
    unsigned int *queue;            // next block of chunks
    int bm_log2;                    // bitmap bits = 1 << bm_log2
    int exact;                      // 1: bit index = column id (ncols <= bitmap bits); 0: one multiplicative hash
    int vals_cap;                   // mask rows up to this long accumulate in shared memory (0: straight into HBM)
    int table;                      // vals_cap > 0: slots of the shared-memory hash (column -> position in the mask row), 2 x vals_cap
    int32_t *spa_slot;              // vals_cap == 0: per-CTA dense map column -> mask position in HBM (ncols entries each, -1 when idle)
    int grab;                       // consecutive chunks per queue grab
    int blk_log2;                   // long B rows are dealt to the warps in blocks of 1 << blk_log2 positions
};

constexpr uint32_t STREAM_LONG_ROW = 1024;      // B rows longer than this are spread over all the warps of the CTA in 128-position trips
constexpr int STREAM_QCAP = 160;                // survivor queue entries per warp: < 32 left over + one trip of 128

__host__ __device__ inline size_t stream_var_smem(int bm_log2, int table, int vals_cap, size_t wsize) {
    const size_t head = ((((size_t)1 << bm_log2) / 8 + (size_t)table * 6 + 7) & ~(size_t)7) + (size_t)vals_cap * (wsize + 1);
    return (head + 15) & ~(size_t)15;
}
template <typename XT> __host__ __device__ inline size_t stream_fixed_smem(int nt) {
    // per-batch A entry arrays + survivor queues (column, B position, batch index of the A entry) + long-row list (entry, first trip)
    return (size_t)nt * (4 + 4 + sizeof(XT)) + (size_t)(nt / 32) * STREAM_QCAP * (8 + 2) + (size_t)nt * (2 + 4) + 64;
}

// One code path, one call site each for the streaming loop and for the survivor drain: the kernel must stay small -- its first
// version inlined the resolve / atomic code at every push (11 k SASS instructions, 176 KB) and lost 2x to instruction fetch.
template <typename XT, typename ZT, int ADD, int MUL>
__global__ void __launch_bounds__(1024, 1) masked_stream_kernel(const StreamArgs sa) {
    typedef typename SlotWord<ZT>::W W;
    const int NT = blockDim.x, NW = NT >> 5;
    const GemmArgs &p = sa.g;
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // layout: [bitmap words][hash keys u32 x table][hash slot u16 x table][vals W x cap][found u8 x cap][s_av][s_bs][s_len][queues][long list]
    const uint32_t bm_words = 1u << (sa.bm_log2 - 5);
    uint32_t *bm = reinterpret_cast<uint32_t *>(smem_raw);
    uint32_t *keys = bm + bm_words;
    uint16_t *slot = reinterpret_cast<uint16_t *>(keys + sa.table);
    W *vals = reinterpret_cast<W *>(smem_raw + (((size_t)bm_words * 4 + (size_t)sa.table * 6 + 7) & ~(size_t)7));
    uint8_t *found = reinterpret_cast<uint8_t *>(vals + sa.vals_cap);
    unsigned char *rest = smem_raw + stream_var_smem(sa.bm_log2, sa.table, sa.vals_cap, sizeof(W));
    const uint32_t tmask = (uint32_t)sa.table - 1u;
    const int hshift = sa.table ? __clz(sa.table) + 1 : 0;
    int32_t *gslot = sa.spa_slot ? sa.spa_slot + (size_t)blockIdx.x * p.ncols : nullptr;
    XT *s_av = reinterpret_cast<XT *>(rest);
    uint32_t *s_bs = reinterpret_cast<uint32_t *>(rest + (size_t)NT * sizeof(XT));
    uint32_t *s_len = s_bs + NT;
    uint32_t *s_ltrip = s_len + NT;                              // long rows: trips before this row (exclusive running sum)
    uint2 *s_q = reinterpret_cast<uint2 *>(s_ltrip + NT);
    uint16_t *s_qe = reinterpret_cast<uint16_t *>(s_q + NW * STREAM_QCAP);
    uint16_t *s_long = s_qe + NW * STREAM_QCAP;
    __shared__ unsigned int s_next, s_nlong, s_ltrips;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const int bm_shift = 32 - sa.bm_log2;
    const bool exact = sa.exact != 0;
    const uint32_t item_len = 1u << sa.blk_log2;               // positions of a long B row one work item covers
    const XT *aval = static_cast<const XT *>(p.a_val), *bval = static_cast<const XT *>(p.b_val);
    W *tw = static_cast<W *>(sa.t_words);
    const W ident = pack_slot<ZT>(accum_init<ZT>(add));
    uint2 *myq = s_q + warp * STREAM_QCAP;
    uint16_t *myqe = s_qe + warp * STREAM_QCAP;

    auto bit_of = [&](uint32_t j) -> uint32_t { return exact ? j : ((j * 2654435761u) >> bm_shift); };

    for (uint32_t w = tid; w < bm_words; w += NT) bm[w] = 0u;
    for (int t = tid; t < sa.table; t += NT) keys[t] = EMPTY_KEY;
    int64_t cur_row = -1; uint32_t ms = 0, me = 0; bool local = false; bool split = false;
    int qn = 0;                                                 // entries in this warp's queue (warp-uniform)
    __syncthreads();

    while (true) {
        if (tid == 0) s_next = atomicAdd(sa.queue, (unsigned int)sa.grab);
        __syncthreads();
        const int64_t c_begin = s_next;
        __syncthreads();
        const bool done = c_begin >= sa.nchunks;
        const int64_t c_end = done ? c_begin + 1 : min(sa.nchunks, c_begin + (int64_t)sa.grab);      // one extra pass to leave the last row
        for (int64_t ch = c_begin; ch < c_end; ++ch) {
            const int64_t row = done ? -1 : sa.chunk_row[ch];
            const uint32_t part = done ? 0u : sa.chunk_idx[ch], nparts = done ? 1u : sa.chunk_cnt[ch];
            if (row != cur_row) {
                // ---- leave the current row: its shared-memory accumulators go to HBM, the bits it set are cleared ...
                if (cur_row >= 0) {
                    const int mlen = (int)(me - ms);
                    if (local) {
                        if (!split) { for (int q = tid; q < mlen; q += NT) { tw[ms + q] = vals[q]; p.t_found[ms + q] = found[q]; } }
                        else for (int q = tid; q < mlen; q += NT) if (found[q]) { atomic_combine<ZT>(&tw[ms + q], unpack_slot<ZT>(vals[q]), add); p.t_found[ms + q] = 1; }
                        for (int t = tid; t < sa.table; t += NT) keys[t] = EMPTY_KEY;
                    }
                    for (uint32_t q = ms + tid; q < me; q += NT) {
                        const uint32_t j = p.m_col[q], b = bit_of(j); bm[b >> 5] = 0u;      // whole words: all their bits are this row's
                        if (gslot) gslot[j] = -1;
                    }
                    __syncthreads();
                }
                cur_row = row;
                // ---- ... and enter the next one: filter bits, hash (or dense map), accumulators
                if (row >= 0) {
                    ms = p.m_ptr[row]; me = p.m_ptr[row + 1]; split = nparts > 1;
                    const int mlen = (int)(me - ms);
                    local = mlen <= sa.vals_cap;
                    if (local) for (int q = tid; q < mlen; q += NT) { vals[q] = ident; found[q] = 0; }
                    for (uint32_t q = ms + tid; q < me; q += NT) {
                        const uint32_t j = p.m_col[q], b = bit_of(j);
                        atomicOr(&bm[b >> 5], 1u << (b & 31));
                        if (local) {                                // mask columns are unique: plain insertion
                            uint32_t h = hash_col(j, hshift);
                            while (atomicCAS(&keys[h], EMPTY_KEY, j) != EMPTY_KEY) h = (h + 1) & tmask;
                            slot[h] = (uint16_t)(q - ms);
                        } else gslot[j] = (int32_t)q;
                    }
                    __syncthreads();
                }
            }
            if (done) break;
            const uint32_t as = p.a_ptr[row], ae = p.a_ptr[row + 1], alen = ae - as;
            const uint32_t c0 = as + (uint32_t)(((uint64_t)alen * part) / nparts), c1 = as + (uint32_t)(((uint64_t)alen * (part + 1)) / nparts);
            for (uint32_t base = c0; base < c1; base += NT) {
                // the batch's A entries: B row range and A value, one per thread
                const uint32_t pa = base + tid;
                uint32_t bs = 0, len = 0; XT av = (XT)1;
                if (pa < c1) {
                    const uint32_t k = __ldg(p.a_col + pa);
                    bs = __ldg(p.b_ptr + k); len = __ldg(p.b_ptr + k + 1) - bs;
                    if (p.need_a) av = gload<XT>(aval + pa);
                }
                if (tid == 0) { s_nlong = 0; s_ltrips = 0; }
                __syncthreads();
                s_bs[tid] = bs; s_len[tid] = len; s_av[tid] = av;
                if (len > STREAM_LONG_ROW) {
                    const uint32_t x = atomicAdd(&s_nlong, 1u);
                    s_long[x] = (uint16_t)tid;
                }
                __syncthreads();
                const int nent = (int)min((uint32_t)NT, c1 - base);
                const int nlong = (int)s_nlong;
                if (tid == 0) {                                   // trips of the long rows, in list order (few rows: serial)
                    uint32_t run = 0;
                    for (int x = 0; x < nlong; ++x) { const int e = s_long[x]; s_ltrip[x] = run; run += (((s_bs[e] & 3u) + s_len[e]) + item_len - 1u) >> sa.blk_log2; }
                    s_ltrips = run;
                }
                __syncthreads();
                // ---- work items of a warp: item < nent = the whole (short) B row of entry `item`; item >= nent = one piece (1 << blk_log2 positions)
                //      of a long row.  One streaming loop serves both.
                const uint32_t nitems = (uint32_t)nent + s_ltrips;
                int lx = 0;                                        // cursor into the long-row list (items come in increasing order)
                for (uint32_t item = warp; ; item += NW) {
                    const bool flush = item >= nitems;            // one last pass per warp: nothing to stream, the queue is emptied
                    int ent = 0; uint32_t s = 0, e = 0;
                    if (!flush) {
                        if (item < (uint32_t)nent) {
                            ent = (int)item;
                            const uint32_t l = s_len[ent];
                            if (l != 0 && l <= STREAM_LONG_ROW) { s = s_bs[ent]; e = s + l; }
                        } else {
                            const uint32_t t = item - (uint32_t)nent;
                            while (lx + 1 < nlong && s_ltrip[lx + 1] <= t) ++lx;
                            ent = s_long[lx];
                            const uint32_t b0 = s_bs[ent], p0 = b0 & ~3u, k = t - s_ltrip[lx];
                            s = max(b0, p0 + k * item_len); e = min(b0 + s_len[ent], p0 + (k + 1u) * item_len);
                        }
                    }
                    // ---- stream positions [s, e): trips of 128 (four consecutive ids per lane, one 128-bit load); the next trip's load is
                    //      issued before this trip is tested.  Trip counts are warp-uniform: every lane takes part in the ballots.
                    uint32_t tb = s & ~3u;
                    uint32_t pb = tb + (uint32_t)lane * 4u;
                    uint4 c = make_uint4(0u, 0u, 0u, 0u);
                    if (pb < e) c = __ldg(reinterpret_cast<const uint4 *>(p.b_col + pb));      // past e: inside B's allocation, valid ids (spgemm_masked)
                    for (; tb < e || (flush && qn > 0); tb += 128u) {
                        const uint32_t pbn = pb + 128u;
                        uint4 cn = make_uint4(0u, 0u, 0u, 0u);
                        if (pbn < e) cn = __ldg(reinterpret_cast<const uint4 *>(p.b_col + pbn));
                        const uint32_t jj[4] = {c.x, c.y, c.z, c.w};
                        bool h[4];
#pragma unroll
                        for (uint32_t i = 0; i < 4; ++i) { const uint32_t b = bit_of(jj[i]); h[i] = ((bm[b >> 5] >> (b & 31u)) & 1u) && pb + i >= s && pb + i < e; }
#pragma unroll
                        for (uint32_t i = 0; i < 4; ++i) {
                            const uint32_t ball = __ballot_sync(0xffffffffu, h[i]);
                            if (h[i]) { const int o = qn + __popc(ball & lt_mask); myq[o] = make_uint2(jj[i], pb + i); myqe[o] = (uint16_t)ent; }
                            qn += __popc(ball);
                        }
                        c = cn; pb = pbn;
                        // ---- survivors: resolved 32 at a time by all lanes (the only place where products are combined)
                        while (qn >= 32 || (flush && qn > 0)) {
                            const int count = min(qn, 32);
                            __syncwarp();
                            if (lane < count) {
                                const uint2 qe = myq[qn - count + lane];
                                const uint32_t j = qe.x;
                                uint32_t lo = 0xffffffffu;
                                if (local) {
                                    uint32_t hh = hash_col(j, hshift);
                                    while (true) {
                                        const uint32_t kk = keys[hh];
                                        if (kk == j) { lo = ms + slot[hh]; break; }
                                        if (kk == EMPTY_KEY) break;                        // a false positive of the filter
                                        hh = (hh + 1) & tmask;
                                    }
                                } else { const int32_t q = gslot[j]; if (q >= 0) lo = (uint32_t)q; }      // one L2 access per survivor
                                if (lo != 0xffffffffu && (p.m_struct || sc_cast(sc_load(p.m_tc, p.m_val, lo), p.m_tc, TC_BOOL).u != 0)) {
                                    const XT bv = p.need_b ? gload<XT>(bval + qe.y) : (XT)1;
                                    const ZT prod = MulApply<XT, ZT>::f(mul, s_av[myqe[qn - count + lane]], bv);
                                    if (local) { atomic_combine<ZT>(&vals[lo - ms], prod, add); found[lo - ms] = 1; }
                                    else { atomic_combine<ZT>(&tw[lo], prod, add); p.t_found[lo] = 1; }
                                }
                            }
                            qn -= count;
                            __syncwarp();
                        }
                    }
                    if (flush) break;
                }
                __syncthreads();                                  // the batch's arrays are about to change (every queue is empty: the flush pass)
            }
        }
        if (done) break;
    }
}
