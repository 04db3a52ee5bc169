// sse_kernel.cu -- stage 1 of the default pipeline (produce).
//
// One persistent warp per connection segment (dynamic ticket):
//   stage    carry tail (HBM, per connection) + new segment bytes -> warp-private shared-memory window
//   split    SWAR/ballot newline scan -> line table            (provider.go:322 ReadBytes('\n'))
//   classify strings.TrimSpace / Contains "[DONE]" / HasPrefix "data: "   (agent.go:178-193), or verbatim (mode P)
//   emit     frame table; a frame that stands in the input arena as it must be sent is a span of it (zero-copy), the others
//            go through the warp-cooperative serializer into the out arena      (agent.go:195 / routes.go:613)
//   items    a stub record + a 16-byte work item per line to decode (lines longer than the window are assembled in the carry
//            slot, past it in line-pool pages, and become work items too); sse_kernel2.cu sorts the items, decodes them
//            (sse_decode_kernel) and resolves early termination (sse_finalize_kernel). An exact `data: [DONE]` line has nothing
//            to decode: its record is written here, final, and it gets no work item.
//   finish   carry update, per-segment result
//
// Pure integer/byte work, no tensor cores.
#include <cuda_runtime.h>
#include <stdint.h>
#include "sse_common.cuh"

namespace {

// ---------------------------------------------------------------- the kernel
// stage 1 of the pipeline (no JSON decoder in this kernel)
#ifndef SSE_V1_MINB
#define SSE_V1_MINB 2
#endif

// ---- SSE_FLAG_COUNTERS (the counting instantiation only)
// Pages held by conn's line-pool chain. Only the warp that has the connection's segment moves its pages during the produce
// launch, so the difference across a call is the pages that call took or returned.
__device__ __forceinline__ uint32_t pool_held(const KParams &P, uint32_t conn) {
    uint32_t n = 0;
    if (P.pool_pages && lane_id() == 0) n = ((volatile PoolChain *)P.pool_chain)[conn].n_pages;
    return __shfl_sync(FULL, n, 0);
}
__device__ __forceinline__ void tally_pages(WarpTally &T, uint32_t before, uint32_t after) {
    T.add(CN_P_POOL_PAGES_TAKEN, after > before ? after - before : 0u);
    T.add(CN_P_POOL_PAGES_RETURNED, before > after ? before - after : 0u);
}
// A line assembled outside the window was completed: its frame (always materialised) and work item, read back from the run
// complete_long_line appended (had_first / last_before: rc before the call).
__device__ __forceinline__ void tally_long_line(const KParams &P, WarpTally &T, const RunChain &rc, bool had_first, uint32_t last_before) {
    uint32_t nf = 0, fl = 0, ni = 0;
    if (lane_id() == 0 && rc.have_first && (!had_first || rc.last_idx != last_before)) {
        const sse_run r = rc.last_idx == SSE_NONE ? rc.first : P.runs[rc.last_idx];   // lane 0 wrote it
        nf = r.frame_count;
        if (nf) fl = P.frames[r.frame_first].len;
        if (r.rec_count && !(P.recs[r.rec_first].flags & SSE_F_DONE_EXACT)) ni = 1;
    }
    nf = __shfl_sync(FULL, nf, 0); fl = __shfl_sync(FULL, fl, 0); ni = __shfl_sync(FULL, ni, 0);
    T.add(CN_P_LINES, 1); T.add(CN_P_LONG_LINES, 1);
    T.add(CN_P_FRAMES_MATERIALISED, nf); T.add(CN_P_BYTES_MATERIALISED, fl); T.add(CN_P_ITEMS, ni);
}

// DEFER: SSE_FLAG_DEFER (its own instantiation: the cold deferral paths do not weigh on the default kernel's registers)
// CNT: SSE_FLAG_COUNTERS (its own instantiation: with CNT = false every counting statement is compiled out)
template <bool DEFER, bool CNT>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, SSE_V1_MINB)
sse_stream_kernel(const __grid_constant__ KParams P) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    CtaSmem &cs = *reinterpret_cast<CtaSmem *>(smem_raw);
    WarpSmem &W = cs.w[threadIdx.x >> 5];
    uint8_t *buf = W.buf;
    const uint32_t lane = lane_id();
    WarpTally T;
    if constexpr (CNT) T.v = 0;

    // tickets are taken one segment ahead: while a segment is processed, the next one's first window is on its way to L2
    uint32_t s_next = 0;
    if (lane == 0) s_next = atomicAdd(&P.ctr->ticket, 1u);
    s_next = __shfl_sync(FULL, s_next, 0);
    for (;;) {
        const uint32_t s = s_next;
        if (s >= P.n_segs) break;
        if constexpr (CNT) T.add(CN_P_SEGMENTS, 1);
        if (lane == 0) s_next = atomicAdd(&P.ctr->ticket, 1u);
        s_next = __shfl_sync(FULL, s_next, 0);
        if (s_next < P.n_segs) {
            const sse_seg nx = P.segs[s_next];
            const uint32_t nb = min(nx.in_len, (uint32_t)BUF);
            for (uint32_t o = lane * 128u; o < nb; o += 32u * 128u) prefetch_l2(P.in + nx.in_off + o);
        }

        const sse_seg seg = P.segs[s];
        uint32_t mode = seg.mode;
        if (mode & SSE_MODE_R) mode |= SSE_MODE_PARSE;
        const uint32_t conn = seg.conn;
        ConnState cst = P.conns[conn];
        uint8_t *slot = P.carry + (size_t)conn * P.carry_slot;
        RunChain rc; rc.have_first = false; rc.last_idx = SSE_NONE; rc.pre = SSE_NONE;
        rc.first.frame_first = rc.first.frame_count = rc.first.rec_first = rc.first.rec_count = 0; rc.first.next = SSE_NONE;
        uint32_t seg_flags = 0;
        if (lane == 0) P.seg_term[s] = SSE_NONE;

        if (cst.flags & (CONN_FINISHED | CONN_DEAD)) {
            if (lane == 0) {
                sse_seg_result r; r.run = rc.first; r.carry_len = cst.carry_len;
                r.flags = (cst.flags & CONN_DEAD) ? SSE_SEG_DEAD : SSE_SEG_FINISHED; r.consumed = seg.in_len;
                P.seg_results[s] = r;
            }
            if constexpr (CNT) T.add(CN_P_SEGMENTS_SKIPPED, 1);
            continue;
        }

        bool in_long = (cst.flags & CONN_LONG) != 0;
        int clen = (int)cst.carry_len;     // bytes in the carry slot
        int pend = 0;                      // bytes at the window front (end at a 16-aligned offset)
        bool carry_front = false;          // the window front holds bytes of an earlier batch (not in this input arena)
        if (!in_long && clen > 0) {
            int A = (clen + 15) & ~15;
            copy_g2s_bytes(buf + (A - clen), slot, clen);
            pend = clen; clen = 0; carry_front = true;
        }
        const bool zero_copy = !(P.flags & SSE_FLAG_COPY_OUT);
        int consumed = 0;
        const int in_len = (int)seg.in_len;
        const uint8_t *src = P.in + seg.in_off;
        // overflow: the segment stops. Without SSE_FLAG_DEFER the batch has failed; with it the rest of the segment is deferred
        // and `consumed` becomes the input-arena offset of the first byte not taken (before seg.in_off: that line starts in the
        // carried tail)
        bool dead = false, overflow = false;

        for (;;) {   // windows
            const int A = (pend + 15) & ~15;
            const int base = A - pend;
            int room = BUF - A;
            int nload = min(in_len - consumed, room);
            {   // 16-byte vector copy HBM -> shared (segment offsets and A are 16-byte aligned)
                const uint4 *g = reinterpret_cast<const uint4 *>(src + consumed);
                uint4 *d = reinterpret_cast<uint4 *>(buf + A);
                int nv = (nload + 15) >> 4;
                for (int i = lane; i < nv; i += 32) d[i] = __ldg(g + i);
            }
            consumed += nload;
            const int fill = A + nload;
            // window position w >= zc_lo holds input byte seg.in_off + ... = w + in_delta (a tail moved to the front is input too)
            const int in_delta = (int)seg.in_off + (consumed - nload) - A;
            const int zc_lo = carry_front ? A : base;
            carry_front = false;
            __syncwarp();
            int pos = base;
            if constexpr (CNT) { T.add(CN_P_WINDOWS, 1); T.add(CN_P_WINDOW_BYTES, (uint32_t)(fill - base)); }

            if (in_long) {
                // still inside a line longer than the window: look for its end only
                int q = -1;
                for (int i0 = base; i0 < fill && q < 0; i0 += 32) {
                    int i = i0 + (int)lane;
                    unsigned m = __ballot_sync(FULL, i < fill && buf[i] == '\n');
                    if (m) q = i0 + __ffs(m) - 1;
                }
                int take = (q < 0) ? (fill - base) : (q - base + 1);
                uint32_t pages = 0;
                if constexpr (DEFER) {      // (the counting instantiation counts pages inside pool_append_defer)
                    const int got = hold_back_defer(P, conn, slot, clen, buf + base, take);
                    if (got < 0) { dead = true; break; }
                    clen += got;
                    __syncwarp();
                    if (got < take) {        // no page for the rest: the segment stops at the first byte the line could not hold
                        consumed = (q < 0 ? fill : q + 1) - (take - got) + in_delta;   // base + got (base is not kept)
                        overflow = true; break;
                    }
                } else {
                    if constexpr (CNT) pages = pool_held(P, conn);
                    const bool held = hold_back(P, conn, slot, clen, buf + base, take);
                    if constexpr (CNT) tally_pages(T, pages, pool_held(P, conn));
                    if (!held) { dead = true; break; }
                    clen += take;
                    __syncwarp();
                }
                if (q < 0) {
                    pend = 0;
                    if (consumed >= in_len) break;
                    continue;
                }
                const bool had_first = rc.have_first;
                const uint32_t last_before = rc.last_idx;
                if constexpr (CNT) pages = pool_held(P, conn);
                const bool completed = complete_long_line<DEFER>(P, rc, conn, slot, clen, mode, s);
                if constexpr (CNT) {
                    tally_pages(T, pages, pool_held(P, conn));
                    if (completed) tally_long_line(P, T, rc, had_first, last_before);
                }
                if (!completed) {
                    consumed = q + in_delta; clen--;   // (SSE_FLAG_DEFER) the segment stops at the line's '\n'
                    overflow = true; break;
                }
                __syncwarp();
                in_long = false; clen = 0; pos = q + 1;
            }

            // ---- rounds of up to LT_MAX lines
            for (;;) {
                if (lane == 0) W.done_cnt = 0;
                __syncwarp();
                // split: newline scan, 16 bytes per lane per step
                int n_lines = 0;
                for (int g0 = pos & ~15; g0 < fill && n_lines < LT_MAX; g0 += 512) {
                    int off = g0 + (int)lane * 16;
                    uint32_t nlm = 0, brm = 0;
                    if (off < fill) {
                        uint4 v = *reinterpret_cast<const uint4 *>(buf + off);
                        nlm = eqmask16(v, 0x0A0A0A0Au);
                        if (mode & SSE_MODE_R) brm = done_candidates16(v);
                        // mask bytes outside [pos, fill)
                        uint32_t valid = 0xFFFFu;
                        if (off < pos) valid &= 0xFFFFu << (pos - off);
                        if (off + 16 > fill) valid &= 0xFFFFu >> (off + 16 - fill);
                        nlm &= valid; brm &= valid;
                    }
                    while (brm) {   // "[DONE]" candidates (agent.go:181)
                        int bpos = off + __ffs(brm) - 1;
                        brm &= brm - 1;
                        if (bpos + 6 <= fill && is_done_at(buf + bpos)) {
                            uint32_t k = atomicAdd(&W.done_cnt, 1u);
                            if (k < DONE_MAX) W.done_pos[k] = (uint16_t)bpos;
                        }
                    }
                    uint32_t cnt = __popc(nlm), pre = cnt;
                    #pragma unroll
                    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(FULL, pre, d); if ((int)lane >= d) pre += t; }
                    uint32_t total = __shfl_sync(FULL, pre, 31);
                    uint32_t idx = (uint32_t)n_lines + pre - cnt;
                    while (nlm) {
                        int bpos = off + __ffs(nlm) - 1;
                        nlm &= nlm - 1;
                        if (idx < LT_MAX) W.lt[idx].nl = (uint16_t)bpos;
                        idx++;
                    }
                    n_lines += (int)total;
                }
                __syncwarp();
                if (n_lines == 0) break;
                if (n_lines > LT_MAX) n_lines = LT_MAX;
                const bool done_ovf = W.done_cnt > DONE_MAX;
                const int n_done = min((int)W.done_cnt, DONE_MAX);

                // classify: one lane per line (2 passes for 64 lines)
                uint32_t my_flen[2] = { 0, 0 }, my_kind[2] = { 0, 0 }, my_parse[2] = { 0, 0 }, my_zc[2] = { 0, 0 }, my_clen[2] = { 0, 0 };
                #pragma unroll
                for (int h = 0; h < 2; h++) {
                    int i = (int)lane + 32 * h;
                    if (i < n_lines) {
                        int ls = (i == 0) ? pos : (int)W.lt[i - 1].nl + 1;
                        int nl = W.lt[i].nl;
                        int a = ls, b = nl + 1;
                        uint32_t kind, parse = 0, zc = 0; int src_s = ls, pay_s = ls, pay_e = ls, flen = 0;
                        if (mode & SSE_MODE_R) {
                            trim_space(buf, a, b);                          // agent.go:178-179
                            bool has_done = false;                          // agent.go:181
                            for (int k = 0; k < n_done; k++) { int d = W.done_pos[k]; if (d >= a && d + 6 <= b) has_done = true; }
                            if (done_ovf && !has_done) for (int k = a; k + 6 <= b; k++) if (is_done_at(buf + k)) { has_done = true; break; }
                            bool pref = is_data_prefix(buf + a, b - a);    // agent.go:186
                            if (has_done) {
                                // swallowed; still decoded for parseStreamingToolCalls (agent.go:182, :377-402)
                                pay_s = pref ? a + 6 : a; pay_e = b;
                                bool exact = pref && (pay_e - pay_s) == 6 && is_done_at(buf + pay_s);   // only `data: [DONE]` ends A6's loop (agent.go:385-396)
                                kind = exact ? K_DONE_EXACT : K_DONE; parse = 1;
                                zc = (zero_copy && pay_s >= zc_lo) ? 1u : 0u;   // split: decoded in place by the decode kernel
                            } else if (pref && b - a > 6) {                  // agent.go:190-197
                                kind = K_EMIT; src_s = a; pay_s = a + 6; pay_e = b; flen = (b - a) + 2; parse = 1;
                                // "data: " + payload + "\n\n" is already what the input holds when nothing was trimmed
                                // at the end and the separator line is empty (the usual upstream framing)
                                zc = (zero_copy && b == nl && a >= zc_lo && nl + 1 < fill && buf[nl + 1] == '\n') ? 1u : 0u;
                            } else kind = K_DROP;
                        } else {
                            kind = K_EMIT; src_s = ls; flen = nl + 1 - ls;   // routes.go:613 verbatim
                            zc = (zero_copy && ls >= zc_lo) ? 1u : 0u;
                            if ((mode & SSE_MODE_PARSE) && is_data_prefix(buf + ls, nl + 1 - ls)) { parse = 1; pay_s = ls + 6; pay_e = nl; }
                        }
                        LineEnt &e = W.lt[i];
                        e.src_s = (uint16_t)src_s; e.pay_s = (uint16_t)pay_s; e.pay_e = (uint16_t)pay_e;
                        // bytes to materialise: a frame that is not a span of the input; also the payload of a swallowed
                        // "[DONE]"-containing line (agent.go:182: still parsed), which the decode kernel reads from an arena
                        const int clen = zc ? 0 : (flen ? flen : (kind == K_DONE ? pay_e - pay_s : 0));
                        e.flen = (uint16_t)flen; e.kind = (uint8_t)kind; e.zc = (uint16_t)zc; e.clen = (uint16_t)clen;
                        my_flen[h] = (uint32_t)flen; my_kind[h] = kind; my_parse[h] = parse; my_zc[h] = zc; my_clen[h] = (uint32_t)clen;
                    }
                }
                // allocate: exclusive prefix (line order) of frame bytes / frame count / rec count
                uint32_t pre_b[2], pre_f[2], pre_r[2], tot_b = 0, tot_f = 0, tot_r = 0;
                #pragma unroll
                for (int h = 0; h < 2; h++) {
                    uint32_t vb = my_clen[h], vf = my_flen[h] ? 1u : 0u, vr = my_parse[h];
                    uint32_t sb = vb, sf = vf, sr = vr;
                    #pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        uint32_t tb = __shfl_up_sync(FULL, sb, d), tf = __shfl_up_sync(FULL, sf, d), tr = __shfl_up_sync(FULL, sr, d);
                        if ((int)lane >= d) { sb += tb; sf += tf; sr += tr; }
                    }
                    pre_b[h] = tot_b + sb - vb; pre_f[h] = tot_f + sf - vf; pre_r[h] = tot_r + sr - vr;
                    tot_b += __shfl_sync(FULL, sb, 31); tot_f += __shfl_sync(FULL, sf, 31); tot_r += __shfl_sync(FULL, sr, 31);
                }
                // every line to decode is a work item; index = rank among this round's items
                uint32_t my_q = 0;
                #pragma unroll
                for (int h = 0; h < 2; h++) my_q += (my_parse[h] && (my_kind[h] == K_EMIT || my_kind[h] == K_DONE)) ? 1u : 0u;
                uint32_t pre_q = my_q;
                #pragma unroll
                for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(FULL, pre_q, d); if ((int)lane >= d) pre_q += t; }
                const uint32_t tot_q = __shfl_sync(FULL, pre_q, 31);
                pre_q -= my_q;
                #pragma unroll
                for (int h = 0; h < 2; h++) {
                    int i = (int)lane + 32 * h;
                    if (i < n_lines && my_parse[h] && (my_kind[h] == K_EMIT || my_kind[h] == K_DONE))
                        W.lt[i].rel = (uint16_t)(pre_q + ((h == 1 && my_parse[0] && (my_kind[0] == K_EMIT || my_kind[0] == K_DONE)) ? 1u : 0u));
                }
                __syncwarp();
                uint32_t ob = 0, qb = 0, fb = 0, rb = 0;
                if (lane == 0) {     // the round's allocation: two 64-bit atomics (Counters: out_bytes | n_items, n_frames | n_recs)
                    const unsigned long long a0 = (unsigned long long)((tot_b + 15u) & ~15u) | ((unsigned long long)tot_q << 32);
                    const unsigned long long a1 = (unsigned long long)tot_f | ((unsigned long long)tot_r << 32);
                    unsigned long long r0 = 0, r1 = 0;
                    if (a0) r0 = atomicAdd(reinterpret_cast<unsigned long long *>(&P.ctr->out_bytes), a0);
                    if (a1) r1 = atomicAdd(reinterpret_cast<unsigned long long *>(&P.ctr->n_frames), a1);
                    ob = (uint32_t)r0; qb = (uint32_t)(r0 >> 32); fb = (uint32_t)r1; rb = (uint32_t)(r1 >> 32);
                }
                ob = __shfl_sync(FULL, ob, 0); fb = __shfl_sync(FULL, fb, 0); rb = __shfl_sync(FULL, rb, 0); qb = __shfl_sync(FULL, qb, 0);
                if constexpr (CNT) T.add(CN_P_ROUNDS, 1);
                if (!DEFER) {
                    if (ob + tot_b + 16 > P.cap_out || fb + tot_f > P.cap_frames || rb + tot_r > P.cap_recs || qb + tot_q > P.cap_items) {
                        // the sort and decode stages still read every work item below cap_items: the round's decode into the sink
                        // record instead of whatever an earlier batch left in the slot
                        empty_items(P, qb, tot_q);
                        if (lane == 0) sse_overflow(P.ctr, SSE_OVF_OUT);
                        overflow = true; break;
                    }
                } else {
                    const bool fits = !(ob + tot_b + 16 > P.cap_out || fb + tot_f > P.cap_frames || rb + tot_r > P.cap_recs ||
                                        qb + tot_q > P.cap_items);
                    const bool need_run = rc.have_first && (tot_f | tot_r) != 0u;
                    if ((!fits || need_run) && !admit_round(P, rc, fits, qb, tot_q, need_run)) {
                        consumed = pos + in_delta;   // the segment stops before this round
                        if constexpr (CNT) T.add(CN_P_DEFERRED_ROUNDS, 1);
                        overflow = true; break;
                    }
                }
                if constexpr (CNT) {
                    uint32_t nzc = 0, nmat = 0, bmat = 0;
                    #pragma unroll
                    for (int h = 0; h < 2; h++)
                        if (my_flen[h]) { if (my_zc[h]) nzc++; else { nmat++; bmat += my_flen[h]; } }
                    T.add(CN_P_LINES, (uint32_t)n_lines); T.add(CN_P_ITEMS, tot_q);
                    T.add(CN_P_FRAMES_ZERO_COPY, __reduce_add_sync(FULL, nzc));
                    T.add(CN_P_FRAMES_MATERIALISED, __reduce_add_sync(FULL, nmat));
                    T.add(CN_P_BYTES_MATERIALISED, __reduce_add_sync(FULL, bmat));
                }
                // frame table
                #pragma unroll
                for (int h = 0; h < 2; h++)
                    if (my_flen[h]) {
                        sse_frame f; f.len = my_flen[h];
                        f.off = my_zc[h] ? P.in_base + (uint32_t)(in_delta + (int)W.lt[(int)lane + 32 * h].src_s) : ob + pre_b[h];
                        P.frames[fb + pre_f[h]] = f;
                    }
                __syncwarp();
                // emit: warp-cooperative serializer, frames back to back in line order (nothing to do when every frame of the
                // round is a span of the input)
                if (tot_b) {
                    uint32_t o = ob;
                    for (int i = 0; i < n_lines; i++) {
                        const LineEnt e = W.lt[i];
                        if (!e.clen) continue;
                        uint8_t *dst = P.out + o;
                        if (!e.flen) copy_s2g_vec(dst, buf + e.pay_s, (int)e.clen);   // payload of a swallowed line (no frame)
                        else if (mode & SSE_MODE_R) {
                            const int body = (int)e.flen - 2;      // "data: " + payload is contiguous in the window
                            copy_s2g_vec(dst, buf + e.src_s, body);
                            if (lane < 2) dst[body + lane] = (uint8_t)'\n';
                        } else copy_s2g_vec(dst, buf + e.src_s, (int)e.flen);
                        o += e.clen;
                    }
                }
                // records, one lane per line: a line to decode gets a stub record and a work item; an exact `data: [DONE]` line
                // (only A6's loop end, agent.go:385-396) gets its final record
                #pragma unroll
                for (int h = 0; h < 2; h++) {
                    int i = (int)lane + 32 * h;
                    if (i < n_lines && my_parse[h]) {
                        const LineEnt e = W.lt[i];
                        const bool exact = my_kind[h] == K_DONE_EXACT, swallowed = my_kind[h] == K_DONE;
                        sse_rec r;
                        r.frame = my_kind[h] == K_EMIT ? fb + pre_f[h] : SSE_NONE; r.flags = exact ? SSE_F_DONE_LINE | SSE_F_DONE_EXACT : 0u;
                        r.content_off = r.content_len = 0; r.tc_first = SSE_NONE; r.tc_count = 0; r.n_choices = 0; r.usage = SSE_NONE;
                        r.payload_len = (uint32_t)(e.pay_e - e.pay_s);
                        P.recs[rb + pre_r[h]] = r;
                        if (exact) continue;
                        uint4 it;
                        // the payload's arena offset: in the input (zero-copy) or where the line was materialised
                        it.x = e.zc ? P.in_base + (uint32_t)(in_delta + (int)e.pay_s) : ob + pre_b[h] + (uint32_t)(e.pay_s - (e.flen ? e.src_s : e.pay_s));
                        it.z = rb + pre_r[h];
                        // scheduling key of the decode kernel's item sort: provider hint x position of the line in its round; the
                        // second decoded line of a round (first content delta, the longest) sorts first: long work early
                        const uint32_t ord = min((uint32_t)e.rel, 7u);
                        const uint32_t cls = ((ord == 1u ? 0u : (ord == 0u ? 1u : ord)) << 2) | (seg.provider & 3u);
                        // bit 31: the line can terminate the stream (emitted, mode R); bit 30: swallowed line (SSE_F_DONE_LINE)
                        it.y = (uint32_t)(e.pay_e - e.pay_s) | (cls << 24) | (swallowed ? 0x40000000u : ((mode & SSE_MODE_R) ? 0x80000000u : 0u));
                        it.w = s;
                        P.items[qb + e.rel] = it;
                    }
                }
                append_run(P, rc, fb, tot_f, rb, tot_r);
                pos = (int)W.lt[n_lines - 1].nl + 1;
                __syncwarp();
            }
            if (overflow) break;

            const int tail = fill - pos;
            // A tail is at most one window (BUF bytes) and sse_init refuses a carry slot shorter than BUF + 16, so the two slot
            // checks below never fail: only a line assembled across windows (in_long, above) can outgrow the slot and go to the pool.
            if (consumed >= in_len) {          // segment exhausted: hold the unterminated tail back
                if (tail > 0) {
                    if (tail > (int)P.carry_slot) { dead = true; break; }
                    copy_s2g_bytes(slot, buf + pos, tail);
                }
                clen = tail;
                break;
            }
            if (tail >= BUF - 32) {            // a whole window without '\n': assemble the line in HBM
                if (tail > (int)P.carry_slot) { dead = true; break; }
                copy_s2g_bytes(slot, buf + pos, tail);
                clen = tail; in_long = true; pend = 0;
                __syncwarp();
                continue;
            }
            // move the tail to the front so that it ends at a 16-byte aligned offset. The window was filled to
            // BUF (more segment bytes remain) and tail < BUF-32, so pos > 32 > destination: the move is toward
            // lower addresses and ascending 32-byte steps (read, sync, write) never clobber unread source bytes.
            {
                const int A2 = (tail + 15) & ~15;
                uint8_t *d = buf + (A2 - tail);
                const uint8_t *sp = buf + pos;
                if (d != sp) {
                    for (int i0 = 0; i0 < tail; i0 += 32) {
                        int i = i0 + (int)lane;
                        uint8_t v = (i < tail) ? sp[i] : (uint8_t)0;
                        __syncwarp();
                        if (i < tail) d[i] = v;
                        __syncwarp();
                    }
                }
                pend = tail;
            }
        }

        if (dead) seg_flags |= SSE_SEG_LINE_TOO_LONG | SSE_SEG_DEAD;
        const bool deferred = DEFER && overflow;
        if (deferred) seg_flags |= SSE_SEG_DEFERRED;
        if (lane == 0) {
            ConnState ns;
            if (deferred) consumed -= (int)P.segs[s].in_off;
            if (deferred && consumed < 0) {
                // deferred at the first line, which starts in the carried tail: the connection is left exactly as it was
                ns = P.conns[conn]; consumed = 0;
            } else {
                ns.carry_len = dead ? 0u : (uint32_t)clen;
                ns.flags = dead ? CONN_DEAD : (in_long ? CONN_LONG : 0u);
                P.conns[conn] = ns;
            }
            sse_seg_result r; r.run = rc.first; r.carry_len = ns.carry_len; r.flags = seg_flags;
            r.consumed = deferred ? (uint32_t)consumed : seg.in_len;
            P.seg_results[s] = r;
        }
        __syncwarp();
    }
    if constexpr (CNT) T.flush(P.cnt, CN_DECODE_FIRST);
}

} // namespace

template <bool DEFER, bool CNT>
static int launch_stream_kernel(const KParams &p, void *stream, int sm_count) {
    static bool attr_set = false;
    static int ctas_per_sm = 0;
    const size_t smem = sizeof(CtaSmem);
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(sse_stream_kernel<DEFER, CNT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
        int n = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, sse_stream_kernel<DEFER, CNT>, WARPS_PER_CTA * 32, smem);
        if (e != cudaSuccess) return (int)e;
        ctas_per_sm = n > 0 ? n : 1;
        attr_set = true;
    }
    int grid = sm_count * ctas_per_sm;   // persistent: one resident wave, warps pull segments by ticket
    int need = (int)((p.n_segs + WARPS_PER_CTA - 1) / WARPS_PER_CTA);
    if (need < grid) grid = need > 0 ? need : 1;
    sse_stream_kernel<DEFER, CNT><<<grid, WARPS_PER_CTA * 32, smem, (cudaStream_t)stream>>>(p);
    return (int)cudaGetLastError();
}

int sse_launch_produce_kernel(const KParams &p, void *stream, int sm_count) {
    if (p.cnt) return (p.flags & SSE_FLAG_DEFER) ? launch_stream_kernel<true, true>(p, stream, sm_count) : launch_stream_kernel<false, true>(p, stream, sm_count);
    return (p.flags & SSE_FLAG_DEFER) ? launch_stream_kernel<true, false>(p, stream, sm_count) : launch_stream_kernel<false, false>(p, stream, sm_count);
}
