// Pileup-counts featuriser on the GPU: the per-base work of calculate_pileup (src/medaka_counts.c:199-372)
// over BAM-packed alignment records (32-bit CIGAR ops, 4-bit sequence), without htslib.
//
// htslib's pileup walks reference positions and, per position, the reads covering it.  Here the loop nest is
// inverted so that it is data-parallel over reads and CIGAR operations:
//   1. plp_walk_kernel   (WARP per read, lanes over CIGAR ops, 32 at a time): reference / query cursor of every op by
//                        warp prefix sums; how insertion runs attach to the reference base before them (htslib's
//                        "peek the next operation" rule, restated in oracle/pileup_oracle.py and pinned on the
//                        reference's real-BAM regression numbers) by a segmented warp scan; the read's coverage as
//                        two entries of a difference array (+1 at its first position in the region, -1 behind its
//                        last); the longest insertion behind every position (atomicMax, insertions only).
//   2. block scans       depth = prefix sum of the difference array; width[pos] = (depth > 0) + longest insertion;
//                        first column of every position = exclusive prefix sum of width.  Three-phase scans (per-block
//                        sums, one small block over the block sums, per-block apply) - no single-block pass over the
//                        region; the (major, minor) arrays come out of the last phase (medaka_counts.c:274-277).
//   3. plp_count_kernel  (thread per op, the warp gangs up on long ops): counts[col][dtype*10 + base] += 1 in the
//                        'acgtACGTdD' feature order (medaka_counts.h:19-30), deletions at minor 0, inserted bases at
//                        minors 1..k (medaka_counts.c:314-357).  32-bit reductions (RED.ADD.U32); widened to the
//                        reference's size_t matrix at the end.
// Read filter: flags and mapQ on the device (medaka_bamiter.c:19-21); tag / read-group / datatype resolution is
// done by the host reader (medaka_b200/bam.py), which hands over a per-read dtype index.
// Reference-skip (N) operations: the read covers the skipped positions (a column exists, nothing is counted there,
// medaka_counts.c:282), and an insertion right behind a skip widens its position's column group but its bases are
// NOT counted (the `continue` at :282 comes before the base loop; the max_ins loop at :259-263 does not look at it).
// All of it is HBM-bound integer/byte work: no tensor cores.  The device scratch is cached per host thread (no
// cudaMalloc on the steady-state path) and nothing synchronises with the host before the final copies.
// Count normalisation (normalise_kernel) lives here too: behind the counts in mdk_pileup_features, on its own in
// mdk_normalise_counts[_dev].
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace mdk {

constexpr int PLP_FILTER_FLAGS = 0x4 | 0x100 | 0x200 | 0x400 | 0x800;   // UNMAP|SECONDARY|QCFAIL|DUP|SUPPLEMENTARY
// 4-bit IUPAC code (+16 if reverse strand) -> index in 'acgtACGTdD' (src/medaka_counts.h:25-30)
__constant__ int8_t c_num2countbase[32] = {-1, 4, 5, -1, 6, -1, -1, -1, 7, -1, -1, -1, -1, -1, -1, -1,
                                           -1, 0, 1, -1, 2, -1, -1, -1, 3, -1, -1, -1, -1, -1, -1, -1};
constexpr int OP_M = 0, OP_I = 1, OP_D = 2, OP_N = 3, OP_S = 4, OP_P = 6, OP_EQ = 7, OP_X = 8;
constexpr uint32_t INS_NOCOUNT = 0x80000000u;   // op_ins flag: the run hangs off a reference skip

__device__ __forceinline__ bool read_passes(uint16_t flag, uint8_t mapq, int min_mapq) {
    return !(flag & PLP_FILTER_FLAGS) && (int)mapq >= min_mapq;
}
__host__ __device__ __forceinline__ bool consumes_ref(int op) { return op == OP_M || op == OP_D || op == OP_N || op == OP_EQ || op == OP_X; }
__host__ __device__ __forceinline__ bool is_match(int op) { return op == OP_M || op == OP_EQ || op == OP_X; }
__host__ __device__ __forceinline__ bool consumes_qry(int op) { return is_match(op) || op == OP_I || op == OP_S; }

// State of the insertion-run scan after an op: kind of the last op that is neither I nor P (0 none yet, 1 consumes the
// reference, 2 reference skip, 3 anything else) and the inserted bases seen since then.  Associative combine: a later
// segment that contains such an op overrides the kind and restarts the sum.
struct RunState {
    uint32_t kind;
    uint32_t ins;
};
__device__ __forceinline__ RunState run_combine(RunState a, RunState b) {
    RunState r;
    r.kind = b.kind ? b.kind : a.kind;
    r.ins = b.kind ? b.ins : a.ins + b.ins;
    return r;
}

// op_ref[k] : reference cursor at the start of op k;  op_qry[k] : query cursor at the start of op k
// op_ins[k] : for an I op attached to reference position op_ref[k] - 1: 1 + the inserted bases before it in its run
//             (| INS_NOCOUNT when the run follows a reference skip); 0 otherwise
// Coverage and longest insertions are only recorded for reads that pass the filter.
__global__ void __launch_bounds__(256) plp_walk_kernel(int64_t n_rec, const int32_t *__restrict__ pos,
                                                       const uint16_t *__restrict__ flag, const uint8_t *__restrict__ mapq,
                                                       int min_mapq, const uint32_t *__restrict__ cigar,
                                                       const int64_t *__restrict__ cigar_off, int32_t start, int32_t end,
                                                       int32_t *__restrict__ op_ref, int32_t *__restrict__ op_qry,
                                                       uint32_t *__restrict__ op_ins, int32_t *__restrict__ cov,
                                                       int32_t *__restrict__ maxins) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (r >= n_rec) return;
    const bool pass = read_passes(flag[r], mapq[r], min_mapq);
    const int64_t k0 = cigar_off[r], k1 = cigar_off[r + 1];
    int32_t x = pos[r], y = 0;                 // cursors at the start of the current chunk of 32 ops
    RunState carry{0u, 0u};
    for (int64_t kb = k0; kb < k1; kb += 32) {
        const int64_t k = kb + lane;
        const bool live = k < k1;
        const uint32_t c = live ? cigar[k] : 0u;
        const int op = live ? (int)(c & 0xF) : OP_P;     // padding consumes nothing and breaks nothing
        const int32_t len = live ? (int32_t)(c >> 4) : 0;
        int32_t dx = consumes_ref(op) ? len : 0;
        int32_t dy = consumes_qry(op) ? len : 0;
        RunState st;
        st.kind = (op == OP_I || op == OP_P) ? 0u : (op == OP_N ? 2u : (consumes_ref(op) ? 1u : 3u));
        st.ins = op == OP_I ? (uint32_t)len : 0u;
        // inclusive warp scans
        int32_t sx = dx, sy = dy;
        RunState ss = st;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t tx = __shfl_up_sync(0xffffffffu, sx, o), ty = __shfl_up_sync(0xffffffffu, sy, o);
            RunState t;
            t.kind = __shfl_up_sync(0xffffffffu, ss.kind, o);
            t.ins = __shfl_up_sync(0xffffffffu, ss.ins, o);
            if (lane >= o) {
                sx += tx;
                sy += ty;
                ss = run_combine(t, ss);
            }
        }
        // state BEFORE this op = carry (+) inclusive state of the previous lane
        RunState before;
        before.kind = __shfl_up_sync(0xffffffffu, ss.kind, 1);
        before.ins = __shfl_up_sync(0xffffffffu, ss.ins, 1);
        if (lane == 0) before = RunState{0u, 0u};
        before = run_combine(carry, before);
        if (live) {
            const int32_t xr = x + sx - dx, yq = y + sy - dy;
            op_ref[k] = xr;
            op_qry[k] = yq;
            uint32_t ins = 0;
            if (op == OP_I && (before.kind == 1u || before.kind == 2u)) {
                ins = (before.ins + 1u) | (before.kind == 2u ? INS_NOCOUNT : 0u);
                const int32_t p = xr - 1;
                if (pass && p >= start && p < end) atomicMax(&maxins[p - start], (int32_t)(before.ins + (uint32_t)len));
            }
            op_ins[k] = ins;
        }
        x += __shfl_sync(0xffffffffu, sx, 31);
        y += __shfl_sync(0xffffffffu, sy, 31);
        RunState last;
        last.kind = __shfl_sync(0xffffffffu, ss.kind, 31);
        last.ins = __shfl_sync(0xffffffffu, ss.ins, 31);
        carry = run_combine(carry, last);
    }
    // the read covers [pos, x): htslib's pileup lists it at every one of those positions (deleted and skipped ones too)
    if (lane == 0 && pass) {
        const int32_t lo = max(pos[r], start), hi = min(x, end);
        if (lo < hi) {
            atomicAdd(&cov[lo - start], 1);
            atomicAdd(&cov[hi - start], -1);
        }
    }
}

// ---------------------------------------------------------------------------------------------- three-phase scans
constexpr int SC_THREADS = 256, SC_PER_THREAD = 8, SC_BLOCK = SC_THREADS * SC_PER_THREAD;   // 2048 positions per block

__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t *total) {
    __shared__ int64_t wsum[SC_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += t;
    }
    __syncthreads();
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    int64_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < SC_THREADS / 32; ++w) {
        if (w < warp) before += wsum[w];
        all += wsum[w];
    }
    if (total) *total = all;
    return before + x - v;
}

// phase 1: per-block sum of the coverage difference array
__global__ void __launch_bounds__(SC_THREADS) plp_sum_cov_kernel(int32_t L, const int32_t *__restrict__ cov,
                                                                 int64_t *__restrict__ blk) {
    const int32_t i0 = blockIdx.x * SC_BLOCK + threadIdx.x * SC_PER_THREAD;
    int64_t s = 0;
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j)
        if (i0 + j < L) s += cov[i0 + j];
    int64_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) blk[blockIdx.x] = total;
}

// phase 2, and the block counts of stitching and variant decoding (decode.cu): exclusive scan of up to a few ten
// thousand block counts, in place, by one block of 1024 threads walking them in 1024-entry strips with the running
// total; counts[n] = the grand total.  Signed: the coverage block sums are sums of a difference array.
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS) scan_blocks_kernel(int64_t *__restrict__ counts, int64_t n) {
    __shared__ int64_t warp_sum[32];
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t s = 0; s < n; s += SCAN_THREADS) {
        const int64_t i = s + threadIdx.x;
        const int64_t v = i < n ? counts[i] : 0;
        int64_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int64_t w = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int64_t y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            warp_sum[lane] = w;                                // inclusive over warps
        }
        __syncthreads();
        const int64_t before = carry + (warp ? warp_sum[warp - 1] : 0) + (x - v);
        if (i < n) counts[i] = before;
        __syncthreads();
        if (threadIdx.x == SCAN_THREADS - 1) carry = before + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[n] = carry;
}

cudaError_t launch_scan_blocks(int64_t *counts, int64_t n, cudaStream_t s) {
    scan_blocks_kernel<<<1, SCAN_THREADS, 0, s>>>(counts, n);
    return cudaGetLastError();
}

// phase 3: depth -> width (kept in `maxins`' array) -> per-block sum of width
__global__ void __launch_bounds__(SC_THREADS) plp_width_kernel(int32_t L, const int32_t *__restrict__ cov,
                                                               const int64_t *__restrict__ blk_cov,
                                                               int32_t *__restrict__ width, int64_t *__restrict__ blk_w) {
    const int32_t i0 = blockIdx.x * SC_BLOCK + threadIdx.x * SC_PER_THREAD;
    int32_t d[SC_PER_THREAD];
    int64_t s = 0;
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j) {
        d[j] = i0 + j < L ? cov[i0 + j] : 0;
        s += d[j];
    }
    int64_t depth = blk_cov[blockIdx.x] + block_exclusive_scan(s, nullptr);
    int64_t w = 0;
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j) {
        depth += d[j];
        if (i0 + j < L) {
            const int32_t wj = depth > 0 ? 1 + width[i0 + j] : 0;     // (width[] holds the longest insertion so far)
            width[i0 + j] = wj;
            w += wj;
        }
    }
    int64_t total;
    block_exclusive_scan(w, &total);
    if (threadIdx.x == 0) blk_w[blockIdx.x] = total;
}

// phase 5 (after the block sums of width have been scanned): first column of every position, position arrays
__global__ void __launch_bounds__(SC_THREADS) plp_columns_kernel(int32_t L, int32_t start, const int32_t *__restrict__ width,
                                                                 const int64_t *__restrict__ blk_w, int64_t max_cols,
                                                                 int64_t *__restrict__ col_off, int64_t *__restrict__ major,
                                                                 int64_t *__restrict__ minor) {
    const int32_t i0 = blockIdx.x * SC_BLOCK + threadIdx.x * SC_PER_THREAD;
    int32_t w[SC_PER_THREAD];
    int64_t s = 0;
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j) {
        w[j] = i0 + j < L ? width[i0 + j] : 0;
        s += w[j];
    }
    int64_t c = blk_w[blockIdx.x] + block_exclusive_scan(s, nullptr);
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j) {
        if (i0 + j < L) {
            col_off[i0 + j] = c;
            for (int32_t m = 0; m < w[j]; ++m) {
                if (c + m < max_cols) {
                    major[c + m] = (int64_t)start + i0 + j;
                    minor[c + m] = m;
                }
            }
            c += w[j];
        }
    }
}

// ---------------------------------------------------------------------------------------------- counting
__device__ __forceinline__ int seq_code(const uint8_t *__restrict__ seq, int64_t base, int32_t q) {
    const uint8_t b = seq[base + (q >> 1)];
    return (q & 1) ? (b & 0xF) : (b >> 4);
}

struct CountOp {
    int32_t lo, hi;        // reference positions [lo, hi) (matches, deletions) or inserted-base indices [0, hi) (lo = 0)
    int32_t x0, q0;        // reference / query cursor at the start of the op
    int64_t col0;          // insertions: first column of the op's bases
    int64_t sbase;         // byte offset of the read's packed sequence
    int32_t fbase;         // 10 * dtype
    int32_t rev;           // 16 when the read is on the reverse strand
    int32_t kind;          // 0 nothing, 1 match, 2 deletion, 3 insertion
};

__device__ __forceinline__ void count_one(const CountOp &o, int32_t i, const uint8_t *__restrict__ seq,
                                          const int64_t *__restrict__ col_off, int32_t start, int F, int64_t max_cols,
                                          uint32_t *__restrict__ counts) {
    if (o.kind == 1) {
        const int bi = c_num2countbase[seq_code(seq, o.sbase, o.q0 + (i - o.x0)) + o.rev];
        const int64_t col = col_off[i - start];
        if (bi >= 0 && col < max_cols) atomicAdd(&counts[col * F + o.fbase + bi], 1u);
    } else if (o.kind == 2) {
        const int64_t col = col_off[i - start];
        if (col < max_cols) atomicAdd(&counts[col * F + o.fbase + (o.rev ? 8 : 9)], 1u);   // rev_del / fwd_del
    } else {
        const int bi = c_num2countbase[seq_code(seq, o.sbase, o.q0 + i) + o.rev];
        if (bi >= 0 && o.col0 + i < max_cols) atomicAdd(&counts[(o.col0 + i) * F + o.fbase + bi], 1u);
    }
}

constexpr int CNT_INLINE = 12;     // bases an op's own thread handles; longer ops are shared out over the warp

__global__ void __launch_bounds__(256) plp_count_kernel(int64_t n_ops, const int32_t *__restrict__ op_rec,
                                                        const uint32_t *__restrict__ cigar, const int32_t *__restrict__ op_ref,
                                                        const int32_t *__restrict__ op_qry, const uint32_t *__restrict__ op_ins,
                                                        const uint16_t *__restrict__ flag, const uint8_t *__restrict__ mapq,
                                                        const uint8_t *__restrict__ dtype, const uint8_t *__restrict__ seq,
                                                        const int64_t *__restrict__ seq_off, int min_mapq, int32_t start,
                                                        int32_t end, int num_dtypes, const int64_t *__restrict__ col_off,
                                                        int64_t max_cols, uint32_t *__restrict__ counts) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const int F = 10 * num_dtypes;
    CountOp o;
    o.kind = 0;
    o.lo = o.hi = 0;
    if (k < n_ops) {
        const int r = op_rec[k];
        const uint16_t fl = flag[r];
        if (read_passes(fl, mapq[r], min_mapq)) {
            const uint32_t c = cigar[k];
            const int op = c & 0xF;
            const int32_t len = (int32_t)(c >> 4);
            o.x0 = op_ref[k];
            o.q0 = op_qry[k];
            o.sbase = seq_off[r];
            o.fbase = 10 * (int)dtype[r];
            o.rev = (fl & 0x10) ? 16 : 0;
            if (is_match(op) || op == OP_D) {
                o.kind = is_match(op) ? 1 : 2;
                o.lo = max(o.x0, start);
                o.hi = min(o.x0 + len, end);
            } else if (op == OP_I) {
                const uint32_t ins = op_ins[k];
                const int32_t p = o.x0 - 1;
                if (ins != 0u && !(ins & INS_NOCOUNT) && p >= start && p < end) {
                    o.kind = 3;
                    o.lo = 0;
                    o.hi = len;
                    o.col0 = col_off[p - start] + (int64_t)(ins & ~INS_NOCOUNT);   // minor 1 + bases before it
                }
            }
            if (o.hi <= o.lo) o.kind = 0;
        }
    }
    const bool big = o.kind != 0 && o.hi - o.lo > CNT_INLINE;
    if (o.kind != 0 && !big)
        for (int32_t i = o.lo; i < o.hi; ++i) count_one(o, i, seq, col_off, start, F, max_cols, counts);
    // long operations (a long match, a multi-kilobase deletion): one after the other, 32 bases per step
    uint32_t todo = __ballot_sync(0xffffffffu, big);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        CountOp w;
        w.lo = __shfl_sync(0xffffffffu, o.lo, src);
        w.hi = __shfl_sync(0xffffffffu, o.hi, src);
        w.x0 = __shfl_sync(0xffffffffu, o.x0, src);
        w.q0 = __shfl_sync(0xffffffffu, o.q0, src);
        w.col0 = __shfl_sync(0xffffffffu, o.col0, src);
        w.sbase = __shfl_sync(0xffffffffu, o.sbase, src);
        w.fbase = __shfl_sync(0xffffffffu, o.fbase, src);
        w.rev = __shfl_sync(0xffffffffu, o.rev, src);
        w.kind = __shfl_sync(0xffffffffu, o.kind, src);
        for (int32_t i = w.lo + lane; i < w.hi; i += 32) count_one(w, i, seq, col_off, start, F, max_cols, counts);
    }
}

__global__ void plp_op_rec_kernel(int64_t n_rec, const int64_t *__restrict__ cigar_off, int32_t *__restrict__ op_rec) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (r >= n_rec) return;
    for (int64_t k = cigar_off[r] + lane; k < cigar_off[r + 1]; k += 32) op_rec[k] = (int32_t)r;
}

__global__ void plp_widen_kernel(int64_t n, const uint32_t *__restrict__ src, uint64_t *__restrict__ dst) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}

// =====================================================================================
// Truth labels of a pileup's columns (HaploidLabelScheme.encode joined to the sample positions, medaka/labels.py:422-484
// and medaka/features.py:979-992) for one truth alignment, without the per-pair dictionary:
//   1. truth_sum_kernel / launch_scan_blocks / truth_ops_kernel: exclusive scans of the reference bases, query bases and
//      reference-consuming ops (length > 0) over the CIGAR, the latter compacting those ops into rstart[j] (reference
//      position of op j's first base) and qstart[j] (query position there), with the end of the alignment as entry
//      n_ref.  Only I and S consume the query between two reference-consuming ops (H and P yield no pairs), so the
//      query-only run behind op j - the insertion columns of its last base - is qstart[j] + (match ? len : 0) ..
//      qstart[j + 1]: a trailing soft clip is the last op's run, a leading one precedes every op and is never looked at.
//   2. truth_label_kernel: one thread per column binary-searches the op holding its major and reads the base there.
// Columns outside [clip_start, clip_end), not covered by the alignment, on a deletion or skip, or beyond their position's
// run get 0, the '*' / padding code.
// =====================================================================================
struct TruthSums {
    int64_t ref, qry, ops;
};

// a thread's SC_PER_THREAD consecutive ops (past the end: 0, an empty M) and their sums
__device__ __forceinline__ TruthSums truth_thread_ops(int64_t i0, int64_t n_ops, const uint32_t *__restrict__ cigar,
                                                      uint32_t (&c)[SC_PER_THREAD]) {
    TruthSums s{0, 0, 0};
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j) {
        c[j] = i0 + j < n_ops ? cigar[i0 + j] : 0u;
        const int op = (int)(c[j] & 0xF);
        const int64_t len = c[j] >> 4;
        if (consumes_ref(op)) {
            s.ref += len;
            s.ops += len > 0;
        }
        if (consumes_qry(op)) s.qry += len;
    }
    return s;
}

// per block of SC_BLOCK ops: blk[0][b], blk[1][b], blk[2][b] = reference bases, query bases, reference-consuming ops
__global__ void __launch_bounds__(SC_THREADS) truth_sum_kernel(int64_t n_ops, const uint32_t *__restrict__ cigar,
                                                               int64_t n_blk, int64_t *__restrict__ blk) {
    uint32_t c[SC_PER_THREAD];
    const TruthSums s = truth_thread_ops(blockIdx.x * (int64_t)SC_BLOCK + threadIdx.x * SC_PER_THREAD, n_ops, cigar, c);
    int64_t tr, tq, tn;
    block_exclusive_scan(s.ref, &tr);
    block_exclusive_scan(s.qry, &tq);
    block_exclusive_scan(s.ops, &tn);
    if (threadIdx.x == 0) {
        blk[blockIdx.x] = tr;
        blk[(n_blk + 1) + blockIdx.x] = tq;
        blk[2 * (n_blk + 1) + blockIdx.x] = tn;
    }
}

// after the three block scans: the compacted reference-consuming ops and the end entry
__global__ void __launch_bounds__(SC_THREADS) truth_ops_kernel(int64_t n_ops, const uint32_t *__restrict__ cigar, int32_t pos,
                                                               int64_t n_blk, const int64_t *__restrict__ blk,
                                                               int64_t *__restrict__ rstart, int64_t *__restrict__ qstart,
                                                               uint8_t *__restrict__ match) {
    const int64_t *blk_ref = blk, *blk_qry = blk + (n_blk + 1), *blk_ops = blk + 2 * (n_blk + 1);
    uint32_t c[SC_PER_THREAD];
    const TruthSums s = truth_thread_ops(blockIdx.x * (int64_t)SC_BLOCK + threadIdx.x * SC_PER_THREAD, n_ops, cigar, c);
    int64_t r = pos + blk_ref[blockIdx.x] + block_exclusive_scan(s.ref, nullptr);
    int64_t q = blk_qry[blockIdx.x] + block_exclusive_scan(s.qry, nullptr);
    int64_t k = blk_ops[blockIdx.x] + block_exclusive_scan(s.ops, nullptr);
#pragma unroll
    for (int j = 0; j < SC_PER_THREAD; ++j) {
        const int op = (int)(c[j] & 0xF);
        const int64_t len = c[j] >> 4;
        if (consumes_ref(op) && len > 0) {
            rstart[k] = r;
            qstart[k] = q;
            match[k] = is_match(op) ? 1 : 0;
            ++k;
        }
        if (consumes_ref(op)) r += len;
        if (consumes_qry(op)) q += len;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        rstart[blk_ops[n_blk]] = pos + blk_ref[n_blk];
        qstart[blk_ops[n_blk]] = blk_qry[n_blk];
    }
}

__global__ void __launch_bounds__(256) truth_label_kernel(int64_t n_cols, const int64_t *__restrict__ major,
                                                          const int64_t *__restrict__ minor, const int64_t *__restrict__ n_ref_dev,
                                                          const int64_t *__restrict__ rstart, const int64_t *__restrict__ qstart,
                                                          const uint8_t *__restrict__ match, const uint8_t *__restrict__ seq,
                                                          int32_t clip_start, int32_t clip_end, int64_t *__restrict__ labels) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_cols) return;
    const int64_t M = major[i], m = minor[i], n_ref = *n_ref_dev;
    int64_t label = 0;
    if (M >= clip_start && M < clip_end) {
        int64_t lo = 0, hi = n_ref;                     // first op starting behind M
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (rstart[mid] <= M) lo = mid + 1; else hi = mid;
        }
        const int64_t j = lo - 1;
        if (j >= 0 && M < rstart[j + 1]) {
            int64_t q = -1;
            if (m == 0) {
                if (match[j]) q = qstart[j] + (M - rstart[j]);
            } else if (m > 0 && M == rstart[j + 1] - 1) {
                const int64_t run = qstart[j] + (match[j] ? rstart[j + 1] - rstart[j] : 0);
                if (m <= qstart[j + 1] - run) q = run + m - 1;
            }
            if (q >= 0) label = c_num2countbase[seq_code(seq, 0, (int32_t)q)] - 3;     // forward A C G T -> 4..7 -> 1..4
        }
    }
    labels[i] = label;
}

// =====================================================================================
// Count normalisation  (CountsFeatureEncoder._post_process_pileup, medaka/features.py:871-935)
// One thread per pileup column.  Algorithmic bytes per column (F=10): read 80 (counts) + 16
// (major, minor), write 40 (features) + 8 (depth) = 144 B.
// =====================================================================================
// index helpers for the per-(dtype, strand) groups of medaka/features.py:647-687:
// feature order per dtype is 'acgtACGTdD' (src/medaka_counts.h:19): reverse = {0,1,2,3,8}, forward = {4,5,6,7,9}
__device__ __forceinline__ bool feat_is_rev(int f10) { return f10 < 4 || f10 == 8; }

__device__ __forceinline__ int64_t lower_bound_major(const int64_t *__restrict__ major, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (major[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <int ND>
__global__ void __launch_bounds__(256) normalise_kernel(const uint64_t *__restrict__ counts,
                                                        const int64_t *__restrict__ major,
                                                        const int64_t *__restrict__ minor, int64_t n, int mode,
                                                        int sym_indels, float *__restrict__ feats,
                                                        int64_t *__restrict__ depth_out) {
    constexpr int F = 10 * ND;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t c[F];
    {
        const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(counts + i * F);
#pragma unroll
        for (int q = 0; q < F / 2; ++q) {
            ulonglong2 v = src[q];
            c[2 * q] = v.x;
            c[2 * q + 1] = v.y;
        }
    }
    const int64_t mn = minor[i];
    // group sums of this column: gs[dt][0] = reverse strand, gs[dt][1] = forward strand
    uint64_t gs_i[ND][2];
#pragma unroll
    for (int dt = 0; dt < ND; ++dt) {
        gs_i[dt][0] = c[dt * 10 + 0] + c[dt * 10 + 1] + c[dt * 10 + 2] + c[dt * 10 + 3] + c[dt * 10 + 8];
        gs_i[dt][1] = c[dt * 10 + 4] + c[dt * 10 + 5] + c[dt * 10 + 6] + c[dt * 10 + 7] + c[dt * 10 + 9];
    }
    uint64_t gs_p[ND][2];      // group sums of the parent (major) column, ORIGINAL counts
    uint64_t del_p[ND][2];     // parent's original deletion counts (needed only if the parent is a minor column)
    int64_t parent_minor = 0;
    if (mn > 0) {
        // np.searchsorted(positions['major'], major, side='left'): first column with this major.  Columns of one
        // major are contiguous with minors counting up from the first one, so the parent is normally mn columns back
        // (two loads to confirm); anything else (a chunk cut inside an insertion run, repeated majors) takes the search.
        const int64_t mj = major[i];
        int64_t j = i - mn;
        if (j < 0 || major[j] != mj || (j > 0 && major[j - 1] == mj)) j = lower_bound_major(major, n, mj);
        parent_minor = minor[j];
        const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(counts + j * F);
        uint64_t p[F];
#pragma unroll
        for (int q = 0; q < F / 2; ++q) {
            ulonglong2 v = src[q];
            p[2 * q] = v.x;
            p[2 * q + 1] = v.y;
        }
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
            gs_p[dt][0] = p[dt * 10 + 0] + p[dt * 10 + 1] + p[dt * 10 + 2] + p[dt * 10 + 3] + p[dt * 10 + 8];
            gs_p[dt][1] = p[dt * 10 + 4] + p[dt * 10 + 5] + p[dt * 10 + 6] + p[dt * 10 + 7] + p[dt * 10 + 9];
            del_p[dt][0] = p[dt * 10 + 8];
            del_p[dt][1] = p[dt * 10 + 9];
        }
    } else {
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
            gs_p[dt][0] = gs_i[dt][0];
            gs_p[dt][1] = gs_i[dt][1];
            del_p[dt][0] = c[dt * 10 + 8];
            del_p[dt][1] = c[dt * 10 + 9];
        }
    }
    // depth = row sum of the parent column's original counts (features.py:889-890)
    uint64_t depth = 0;
#pragma unroll
    for (int dt = 0; dt < ND; ++dt) depth += gs_p[dt][0] + gs_p[dt][1];
    if (depth_out) depth_out[i] = (int64_t)depth;

    if (sym_indels && mn > 0) {
        // features.py:892-908: reads spanning the insertion site without the insertion count as deletions
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
            c[dt * 10 + 8] = gs_p[dt][0] - gs_i[dt][0];   // uint64 wrap-around like numpy
            c[dt * 10 + 9] = gs_p[dt][1] - gs_i[dt][1];
        }
    }
    float out[F];
    if (mode == MDK_NORM_TOTAL) {
        const double d = (double)(depth > 1 ? depth : 1);
#pragma unroll
        for (int f = 0; f < F; ++f) out[f] = __double2float_rn((double)c[f] / d);   // f64 divide then cast (features.py:914,926)
    } else if (mode == MDK_NORM_FWD_REV) {
        // features.py:915-923: per (dtype, strand) depth, recomputed from the (possibly sym_indels-modified)
        // counts; minor columns take their parent's group depth.
#pragma unroll
        for (int dt = 0; dt < ND; ++dt) {
#pragma unroll
            for (int st = 0; st < 2; ++st) {
                uint64_t g;
                if (mn > 0) {
                    g = gs_p[dt][st];
                    // parent itself a minor column (chunk cut inside an insertion run): its own deletion
                    // slot was overwritten by the sym_indels fill (with gs_p - gs_p = 0)
                    if (sym_indels && parent_minor > 0) g -= del_p[dt][st];
                } else {
                    g = gs_i[dt][st];
                }
                const double d = (double)(g > 1 ? g : 1);
#pragma unroll
                for (int b = 0; b < 10; ++b) {
                    if (feat_is_rev(b) == (st == 0)) out[dt * 10 + b] = __double2float_rn((double)c[dt * 10 + b] / d);
                }
            }
        }
    } else {
#pragma unroll
        for (int f = 0; f < F; ++f) out[f] = (float)c[f];
    }
    float2 *dst = reinterpret_cast<float2 *>(feats + i * F);
#pragma unroll
    for (int q = 0; q < F / 2; ++q) dst[q] = make_float2(out[2 * q], out[2 * q + 1]);
}

static cudaError_t launch_normalise(const uint64_t *counts, const int64_t *major, const int64_t *minor, int64_t n,
                             int num_dtypes, int mode, int sym_indels, float *feats, int64_t *depth,
                             cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    const int threads = 256;
    const unsigned blocks = (unsigned)((n + threads - 1) / threads);
    switch (num_dtypes) {
        case 1: normalise_kernel<1><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        case 2: normalise_kernel<2><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        case 3: normalise_kernel<3><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        case 4: normalise_kernel<4><<<blocks, threads, 0, s>>>(counts, major, minor, n, mode, sym_indels, feats, depth); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}


// =========================================================================================================
// Read-level featuriser: calculate_read_alignment (src/medaka_read_matrix.c:277-615) - one int8 feature vector per
// (pileup column, read row): base 1..4 / 5 = deletion, base quality, strand, mapping quality [, dwell][, haplotype]
// [, datatype].  The column structure is the counts featuriser's (same walk / scans); which ROW a read occupies is the
// reference's sequential greedy bookkeeping and is replayed on the host (rm_assign_rows); the cells are filled on the
// device, thread per CIGAR operation like plp_count_kernel.
// =========================================================================================================
// 4-bit IUPAC code -> 1..4 for ACGT, -1 otherwise (src/medaka_read_matrix.h:41-46)
__constant__ int8_t c_num2countbase_symm[16] = {-1, 1, 2, -1, 3, -1, -1, -1, 4, -1, -1, -1, -1, -1, -1, -1};
constexpr int RM_DEL_VAL = 5;          // src/medaka_read_matrix.h:38

struct RmArgs {
    const int32_t *op_rec, *op_ref, *op_qry;
    const uint32_t *cigar, *op_ins;
    const int64_t *cigar_off;
    const uint16_t *flag;
    const uint8_t *mapq, *dtype, *seq, *qual;
    const int64_t *seq_off, *qual_off;
    const int8_t *dwell;               // per base (qual_off indexing), 0 where the read has no usable move table; or null
    const uint8_t *has_dwell;          // per read
    const uint8_t *hap;                // per read; or null
    const int32_t *row;                // per read: row of the matrix, -1 = not placed
    const int32_t *width;
    const int64_t *col_off;
    int32_t start, end;
    int32_t n_rows, featlen, f_dwell, f_hap, f_dtype;     // feature slots (-1 = absent)
    int64_t max_cols;
    int8_t *matrix;
};

__device__ __forceinline__ void rm_cell(const RmArgs &a, int64_t col, int row, int base, int qual, int strand, int mq,
                                        int dwell, bool write_dwell, int hap, int dt) {
    if (col >= a.max_cols) return;
    int8_t *c = a.matrix + (col * a.n_rows + row) * a.featlen;
    c[0] = (int8_t)base;
    c[1] = (int8_t)qual;
    c[2] = (int8_t)strand;
    c[3] = (int8_t)mq;
    if (a.f_dwell >= 0 && write_dwell) c[a.f_dwell] = (int8_t)dwell;
    if (a.f_hap >= 0) c[a.f_hap] = (int8_t)hap;
    if (a.f_dtype >= 0) c[a.f_dtype] = (int8_t)dt;
}

struct RmOp {
    int32_t lo, hi, x0, q0, len;
    int32_t tail_ins;      // inserted bases hanging off the op's last reference position (counted runs only)
    int64_t col0, sbase, qbase;
    int32_t row, strand, mq, hap, dt, hasdw;
    int32_t kind;          // 0 nothing, 1 match, 2 deletion, 3 insertion
};

__device__ __forceinline__ void rm_one(const RmArgs &a, const RmOp &o, int32_t i) {
    if (o.kind == 3) {
        const int32_t q = o.q0 + i;
        const int base = c_num2countbase_symm[seq_code(a.seq, o.sbase, q)];
        rm_cell(a, o.col0 + i, o.row, base, a.qual[o.qbase + q], o.strand, o.mq, a.dwell ? a.dwell[o.qbase + q] : 0,
                o.hasdw != 0, o.hap, o.dt);
        return;
    }
    const int64_t col = a.col_off[i - a.start];
    const int32_t w = a.width[i - a.start];
    int32_t own = 0;                                    // minors this read fills with its own inserted bases
    if (i == o.x0 + o.len - 1) own = o.tail_ins;
    if (o.kind == 1) {
        const int32_t q = o.q0 + (i - o.x0);
        const int base = c_num2countbase_symm[seq_code(a.seq, o.sbase, q)];
        rm_cell(a, col, o.row, base, a.qual[o.qbase + q], o.strand, o.mq, a.dwell ? a.dwell[o.qbase + q] : 0, o.hasdw != 0,
                o.hap, o.dt);
    } else {
        rm_cell(a, col, o.row, RM_DEL_VAL, -1, o.strand, o.mq, -1, true, o.hap, o.dt);       // :473-494
    }
    for (int32_t m = own + 1; m < w; ++m)                                                    // :527-553
        rm_cell(a, col + m, o.row, RM_DEL_VAL, -1, o.strand, o.mq, -1, true, o.hap, o.dt);
}

__global__ void __launch_bounds__(256) plp_fill_kernel(int64_t n_ops, RmArgs a, int min_mapq) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    RmOp o;
    o.kind = 0;
    o.lo = o.hi = 0;
    if (k < n_ops) {
        const int r = a.op_rec[k];
        const uint16_t fl = a.flag[r];
        const int32_t row = a.row[r];
        if (row >= 0 && row < a.n_rows && read_passes(fl, a.mapq[r], min_mapq)) {
            const uint32_t c = a.cigar[k];
            const int op = c & 0xF;
            o.len = (int32_t)(c >> 4);
            o.x0 = a.op_ref[k];
            o.q0 = a.op_qry[k];
            o.sbase = a.seq_off[r];
            o.qbase = a.qual_off[r];
            o.row = row;
            o.strand = (fl & 0x10) ? -1 : 1;
            o.mq = (int8_t)a.mapq[r];
            o.hap = a.hap ? a.hap[r] : 0;
            o.dt = a.dtype[r];
            o.hasdw = a.has_dwell ? a.has_dwell[r] : 0;
            o.tail_ins = 0;
            if (is_match(op) || op == OP_D) {
                o.kind = is_match(op) ? 1 : 2;
                o.lo = max(o.x0, a.start);
                o.hi = min(o.x0 + o.len, a.end);
                // insertion run behind the op's last position (htslib's "peek the next operation", I and P only)
                const int64_t k1 = a.cigar_off[r + 1];
                for (int64_t j = k + 1; j < k1; ++j) {
                    const uint32_t cj = a.cigar[j];
                    const int opj = cj & 0xF;
                    if (opj == OP_I) o.tail_ins += (int32_t)(cj >> 4);
                    else if (opj != OP_P) break;
                }
            } else if (op == OP_I) {
                const uint32_t ins = a.op_ins[k];
                const int32_t p = o.x0 - 1;
                if (ins != 0u && !(ins & INS_NOCOUNT) && p >= a.start && p < a.end) {
                    o.kind = 3;
                    o.lo = 0;
                    o.hi = o.len;
                    o.col0 = a.col_off[p - a.start] + (int64_t)(ins & ~INS_NOCOUNT);
                }
            }
            if (o.hi <= o.lo) o.kind = 0;
        }
    }
    const bool big = o.kind != 0 && o.hi - o.lo > CNT_INLINE;
    if (o.kind != 0 && !big)
        for (int32_t i = o.lo; i < o.hi; ++i) rm_one(a, o, i);
    uint32_t todo = __ballot_sync(0xffffffffu, big);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        RmOp w;
        w.lo = __shfl_sync(0xffffffffu, o.lo, src);
        w.hi = __shfl_sync(0xffffffffu, o.hi, src);
        w.x0 = __shfl_sync(0xffffffffu, o.x0, src);
        w.q0 = __shfl_sync(0xffffffffu, o.q0, src);
        w.len = __shfl_sync(0xffffffffu, o.len, src);
        w.tail_ins = __shfl_sync(0xffffffffu, o.tail_ins, src);
        w.col0 = __shfl_sync(0xffffffffu, o.col0, src);
        w.sbase = __shfl_sync(0xffffffffu, o.sbase, src);
        w.qbase = __shfl_sync(0xffffffffu, o.qbase, src);
        w.row = __shfl_sync(0xffffffffu, o.row, src);
        w.strand = __shfl_sync(0xffffffffu, o.strand, src);
        w.mq = __shfl_sync(0xffffffffu, o.mq, src);
        w.hap = __shfl_sync(0xffffffffu, o.hap, src);
        w.dt = __shfl_sync(0xffffffffu, o.dt, src);
        w.hasdw = __shfl_sync(0xffffffffu, o.hasdw, src);
        w.kind = __shfl_sync(0xffffffffu, o.kind, src);
        for (int32_t i = w.lo + lane; i < w.hi; i += 32) rm_one(a, w, i);
    }
}

// Column structure of a region, shared by the counts and the read-level featurisers and only enqueued on s: op_rec /
// op_ref / op_qry / op_ins / width / col_off in the SCRATCH blob, major / minor written, the number of columns left on
// the device at n_cols for the caller to read once its own kernels are queued.  tail_words more 32-bit words of the
// scratch, zeroed, are the caller's (the counts' accumulator).
struct ColumnPlan {
    int32_t *op_rec, *op_ref, *op_qry, *width;
    uint32_t *op_ins, *tail;
    int64_t *col_off;
    const int64_t *n_cols;
};
static int plan_columns(int64_t n_rec, const Records &d, int64_t n_ops, int32_t start, int32_t end, int min_mapq,
                        int64_t max_cols, int64_t *major, int64_t *minor, size_t tail_words, ColumnPlan *plan,
                        cudaStream_t s) {
    const int32_t L = end - start;
    const int64_t n_blk = (L + SC_BLOCK - 1) / SC_BLOCK;
    Staging sc(Blob::SCRATCH, "pileup column plan");
    int32_t *cov;
    int64_t *blk_cov, *blk_w;
    sc.take(&plan->op_rec, n_ops);
    sc.take(&plan->op_ref, n_ops);
    sc.take(&plan->op_qry, n_ops);
    sc.take(&plan->op_ins, n_ops);
    sc.take(&cov, L + 1);
    sc.take(&plan->width, L);
    sc.take(&plan->col_off, L);
    sc.take(&blk_cov, n_blk + 1);
    sc.take(&blk_w, n_blk + 1);
    sc.take(&plan->tail, tail_words);
    if (!sc.alloc()) return sc.result();
    // cov and width are adjacent: one memset
    MDK_CUDA(cudaMemsetAsync(cov, 0, (size_t)((uint8_t *)(plan->width + L) - (uint8_t *)cov), s));
    if (tail_words) MDK_CUDA(cudaMemsetAsync(plan->tail, 0, tail_words * 4, s));
    const unsigned wb = (unsigned)((n_rec * 32 + 255) / 256);
    plp_op_rec_kernel<<<wb, 256, 0, s>>>(n_rec, d.cigar_off, plan->op_rec);
    plp_walk_kernel<<<wb, 256, 0, s>>>(n_rec, d.pos, d.flag, d.mapq, min_mapq, d.cigar, d.cigar_off, start, end,
                                       plan->op_ref, plan->op_qry, plan->op_ins, cov, plan->width);
    plp_sum_cov_kernel<<<(unsigned)n_blk, SC_THREADS, 0, s>>>(L, cov, blk_cov);
    MDK_CUDA(launch_scan_blocks(blk_cov, n_blk, s));
    plp_width_kernel<<<(unsigned)n_blk, SC_THREADS, 0, s>>>(L, cov, blk_cov, plan->width, blk_w);
    MDK_CUDA(launch_scan_blocks(blk_w, n_blk, s));
    plp_columns_kernel<<<(unsigned)n_blk, SC_THREADS, 0, s>>>(L, start, plan->width, blk_w, max_cols, plan->col_off,
                                                              major, minor);
    MDK_CUDA(cudaGetLastError());
    plan->n_cols = blk_w + n_blk;
    return MDK_OK;
}

// Counts of a region (device pointers in, device pointers out).  Returns the number of columns through *n_cols_host;
// if it exceeds max_cols the outputs are incomplete and the caller re-runs with a larger buffer (the reference's
// enlarge_plp_data, medaka_counts.c:266-271).
int pileup_counts_dev(int64_t n_rec, const Records &d, int64_t n_ops, int32_t start, int32_t end, int num_dtypes,
                             int min_mapq, int64_t max_cols, uint64_t *counts, int64_t *major, int64_t *minor,
                             int64_t *n_cols_host, cudaStream_t s) {
    *n_cols_host = 0;
    if (end <= start || n_rec == 0 || n_ops == 0) return MDK_OK;
    const int F = 10 * num_dtypes;
    ColumnPlan plan;
    int rc = plan_columns(n_rec, d, n_ops, start, end, min_mapq, max_cols, major, minor, (size_t)max_cols * F, &plan, s);
    if (rc) return rc;
    if (max_cols > 0) {
        plp_count_kernel<<<(unsigned)((n_ops + 255) / 256), 256, 0, s>>>(
            n_ops, plan.op_rec, d.cigar, plan.op_ref, plan.op_qry, plan.op_ins, d.flag, d.mapq, d.dtype, d.seq, d.seq_off,
            min_mapq, start, end, num_dtypes, plan.col_off, max_cols, plan.tail);
        const int64_t n_out = max_cols * F;
        plp_widen_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, s>>>(n_out, plan.tail, counts);
    }
    MDK_CUDA(cudaGetLastError());
    MDK_CUDA(cudaMemcpyAsync(n_cols_host, plan.n_cols, 8, cudaMemcpyDeviceToHost, s));
    MDK_CUDA(cudaStreamSynchronize(s));
    return MDK_OK;
}

static int read_matrix_dev(int64_t n_rec, const Records &d, int64_t n_ops, const uint8_t *qual, const int64_t *qual_off,
                           const int8_t *dwell, const uint8_t *has_dwell, const uint8_t *hap, const int32_t *row,
                           int32_t start, int32_t end, int min_mapq, int n_rows, int featlen, int f_dwell, int f_hap,
                           int f_dtype, int64_t max_cols, int8_t *matrix, int64_t *major, int64_t *minor,
                           int64_t *n_cols_host, cudaStream_t s) {
    *n_cols_host = 0;
    if (end <= start || n_rec == 0 || n_ops == 0) return MDK_OK;
    ColumnPlan plan;
    int rc = plan_columns(n_rec, d, n_ops, start, end, min_mapq, max_cols, major, minor, 0, &plan, s);
    if (rc) return rc;
    MDK_CUDA(cudaMemcpyAsync(n_cols_host, plan.n_cols, 8, cudaMemcpyDeviceToHost, s));
    MDK_CUDA(cudaStreamSynchronize(s));
    if (*n_cols_host > max_cols || n_rows <= 0 || max_cols == 0) return MDK_OK;      // caller retries / nothing to fill
    MDK_CUDA(cudaMemsetAsync(matrix, 0, (size_t)(*n_cols_host) * n_rows * featlen, s));
    RmArgs a;
    a.op_rec = plan.op_rec; a.op_ref = plan.op_ref; a.op_qry = plan.op_qry; a.cigar = d.cigar; a.op_ins = plan.op_ins;
    a.cigar_off = d.cigar_off; a.flag = d.flag; a.mapq = d.mapq; a.dtype = d.dtype; a.seq = d.seq; a.qual = qual;
    a.seq_off = d.seq_off; a.qual_off = qual_off; a.dwell = dwell; a.has_dwell = has_dwell; a.hap = hap; a.row = row;
    a.width = plan.width; a.col_off = plan.col_off; a.start = start; a.end = end; a.n_rows = n_rows; a.featlen = featlen;
    a.f_dwell = f_dwell; a.f_hap = f_hap; a.f_dtype = f_dtype; a.max_cols = max_cols; a.matrix = matrix;
    plp_fill_kernel<<<(unsigned)((n_ops + 255) / 256), 256, 0, s>>>(n_ops, a, min_mapq);
    MDK_CUDA(cudaGetLastError());
    MDK_CUDA(cudaStreamSynchronize(s));
    return MDK_OK;
}

}  // namespace mdk

// ---------------------------------------------------------------------------------------------------------
// Host side of the read-level featuriser: the reference's row bookkeeping (medaka_read_matrix.c:329-464), replayed over
// the emitted positions of the region.  Sequential by definition (a new read takes the first row whose previous read
// ended at least five positions ago, in pileup order), O(positions + reads x rows) - microseconds per 100 kb.
namespace mdk {

struct RmHostRead {
    int32_t first_active = -1;     // first region position where the read is listed and is not inside a reference skip
    int64_t ref_end = 0;           // pos + aligned length over M, D, =, X (NOT N: aligned_ref_pos_from_cigar, :258-273)
};

static int8_t rm_clamp_dwell(uint32_t d) { return (int8_t)(d < 127u ? d : 127u); }

// aux walk: finds the `mv` move table (B array) and the `HP` integer of one record
static void rm_scan_aux(const uint8_t *a, int64_t n, const uint8_t **mv, char *mv_type, uint32_t *mv_len, int *hp) {
    *mv = nullptr; *mv_len = 0; *mv_type = 0; *hp = 0;
    int64_t i = 0;
    auto isize = [](char t) { return t == 'c' || t == 'C' || t == 'A' ? 1 : (t == 's' || t == 'S' ? 2 : (t == 'i' || t == 'I' || t == 'f' ? 4 : 0)); };
    while (i + 3 <= n) {
        const char t0 = (char)a[i], t1 = (char)a[i + 1], ty = (char)a[i + 2];
        i += 3;
        if (ty == 'Z' || ty == 'H') {
            while (i < n && a[i]) ++i;
            ++i;
        } else if (ty == 'B') {
            if (i + 5 > n) return;
            const char sub = (char)a[i];
            const uint32_t cnt = (uint32_t)a[i + 1] | ((uint32_t)a[i + 2] << 8) | ((uint32_t)a[i + 3] << 16) | ((uint32_t)a[i + 4] << 24);
            const int w = isize(sub);
            if (!w) return;
            if (t0 == 'm' && t1 == 'v') { *mv = a + i + 5; *mv_type = sub; *mv_len = cnt; }
            i += 5 + (int64_t)cnt * w;
        } else {
            const int w = isize(ty);
            if (!w) return;
            if (t0 == 'H' && t1 == 'P' && i + w <= n) {
                int64_t v = 0;
                switch (ty) {
                    case 'c': v = (int8_t)a[i]; break;
                    case 'C': v = a[i]; break;
                    case 's': v = (int16_t)(a[i] | (a[i + 1] << 8)); break;
                    case 'S': v = (uint16_t)(a[i] | (a[i + 1] << 8)); break;
                    case 'i': case 'I': v = (int32_t)((uint32_t)a[i] | ((uint32_t)a[i + 1] << 8) | ((uint32_t)a[i + 2] << 16) | ((uint32_t)a[i + 3] << 24)); break;
                    default: break;
                }
                *hp = (int)(v & 0xFF);      // uint8_t haplotype (:414)
            }
            i += w;
        }
    }
}

static int64_t rm_mv_at(const uint8_t *mv, char type, uint32_t i) {
    switch (type) {
        case 'c': return (int8_t)mv[i];
        case 'C': return mv[i];
        case 's': return (int16_t)(mv[2 * i] | (mv[2 * i + 1] << 8));
        case 'S': return (uint16_t)(mv[2 * i] | (mv[2 * i + 1] << 8));
        default: return (int32_t)((uint32_t)mv[4 * i] | ((uint32_t)mv[4 * i + 1] << 8) | ((uint32_t)mv[4 * i + 2] << 16) | ((uint32_t)mv[4 * i + 3] << 24));
    }
}

// calculate_dwells (:154-213).  Returns false (no dwell channel for this read) when the table is absent or does not fit.
static bool rm_dwells(const uint8_t *mv, char type, uint32_t mv_len, bool reverse, int32_t length, int8_t *out) {
    if (!mv || length <= 0) return false;
    int64_t qpos = 0;
    if (reverse) {
        uint32_t dwell = 0;
        for (uint32_t i = mv_len ? mv_len - 1 : 0; i > 0; --i) {
            ++dwell;
            if (rm_mv_at(mv, type, i) == 1) {
                if (qpos >= length) return false;
                out[qpos++] = rm_clamp_dwell(dwell);
                dwell = 0;
            }
        }
    } else {
        uint32_t dwell = 1;
        for (uint32_t i = 2; i < mv_len; ++i) {
            if (rm_mv_at(mv, type, i) == 1) {
                if (qpos >= length) return false;
                out[qpos++] = rm_clamp_dwell(dwell);
                dwell = 0;
            }
            ++dwell;
        }
        if (qpos >= length) return false;     // (the reference stores one past its array here)
        out[qpos] = rm_clamp_dwell(dwell);
    }
    return true;
}

// The record arrays are laid out first, and their device copies named in *d; the caller's own arrays go behind them.
static void stage_records(Staging &st, int64_t n_rec, const Records &h, Records *d) {
    st.in(&d->pos, h.pos, n_rec);
    st.in(&d->flag, h.flag, n_rec);
    st.in(&d->mapq, h.mapq, n_rec);
    st.in(&d->dtype, h.dtype, n_rec);
    st.in(&d->cigar, h.cigar, h.cigar_off[n_rec]);
    st.in(&d->cigar_off, h.cigar_off, n_rec + 1);
    st.in(&d->seq, h.seq, h.seq_off[n_rec]);
    st.in(&d->seq_off, h.seq_off, n_rec + 1);
}

// The normalisation switches of mdk_pileup_features / mdk_normalise_counts and where the features go
struct Normalise {
    int mode, sym_indels;
    float *feats;
    int64_t *depth;
};

// mdk_pileup_counts (norm == nullptr: the counts come back) and mdk_pileup_features (the counts are normalised on the
// device and the features come back), once their arguments are checked.
static int pileup_host(const char *what, int device, int64_t n_rec, const Records &h, int32_t start, int32_t end,
                       int num_dtypes, int min_mapq, int64_t max_cols, uint64_t *counts_out, const Normalise *norm,
                       int64_t *major_out, int64_t *minor_out, int64_t *n_cols_out) {
    MDK_CUDA(cudaSetDevice(device));
    const int F = 10 * num_dtypes;
    Staging st(Blob::STAGING, what);
    Records d;
    stage_records(st, n_rec, h, &d);
    uint64_t *d_counts;
    int64_t *d_major, *d_minor, *d_depth = nullptr;
    float *d_feats = nullptr;
    st.take(&d_counts, max_cols * F);
    st.take(&d_major, max_cols);
    st.take(&d_minor, max_cols);
    if (norm) {
        st.take(&d_feats, max_cols * F);
        st.take(&d_depth, max_cols);
    }
    if (!st.alloc()) return st.result();
    int rc = pileup_counts_dev(n_rec, d, h.cigar_off[n_rec], start, end, num_dtypes, min_mapq, max_cols, d_counts, d_major,
                               d_minor, n_cols_out, 0);
    if (rc) return rc;
    const int64_t n = *n_cols_out;
    if (n > max_cols) {
        set_error(std::string(what) + ": output buffers too small (see *n_cols_out)");
        return MDK_ERR_NOMEM;
    }
    if (norm) {
        st.check(launch_normalise(d_counts, d_major, d_minor, n, num_dtypes, norm->mode, norm->sym_indels, d_feats, d_depth,
                                  0));
        st.out(norm->feats, d_feats, n * F);
        if (norm->depth) st.out(norm->depth, d_depth, n);
    } else {
        st.out(counts_out, d_counts, n * F);
    }
    st.out(major_out, d_major, n);
    st.out(minor_out, d_minor, n);
    return st.result();
}

}  // namespace mdk

using namespace mdk;

extern "C" {

int mdk_normalise_counts_dev(int device, const uint64_t *counts_dev, const int64_t *major_dev,
                             const int64_t *minor_dev, int64_t n, int32_t num_dtypes, int32_t mode,
                             int32_t sym_indels, float *feats_out_dev, int64_t *depth_out_dev) {
    MDK_REQUIRE(n >= 0, MDK_ERR_ARG, "normalise_counts: n < 0");
    MDK_REQUIRE(num_dtypes >= 1 && num_dtypes <= 4, MDK_ERR_UNSUPPORTED, "normalise_counts: 1..4 dtypes supported");
    MDK_REQUIRE(mode >= MDK_NORM_TOTAL && mode <= MDK_NORM_NONE, MDK_ERR_ARG, "normalise_counts: unknown mode");
    if (n == 0) return MDK_OK;
    MDK_REQUIRE(counts_dev && major_dev && minor_dev && feats_out_dev, MDK_ERR_ARG, "normalise_counts: NULL pointer");
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(launch_normalise(counts_dev, major_dev, minor_dev, n, num_dtypes, mode, sym_indels, feats_out_dev,
                              depth_out_dev, 0));
    return MDK_OK;
}

int mdk_normalise_counts(int device, const uint64_t *counts, const int64_t *major, const int64_t *minor, int64_t n,
                         int32_t num_dtypes, int32_t mode, int32_t sym_indels, float *feats_out,
                         int64_t *depth_out) {
    MDK_REQUIRE(n >= 0, MDK_ERR_ARG, "normalise_counts: n < 0");
    MDK_REQUIRE(num_dtypes >= 1 && num_dtypes <= 4, MDK_ERR_UNSUPPORTED, "normalise_counts: 1..4 dtypes supported");
    if (n == 0) return MDK_OK;
    MDK_REQUIRE(counts && major && minor && feats_out, MDK_ERR_ARG, "normalise_counts: NULL pointer");
    MDK_CUDA(cudaSetDevice(device));
    const size_t F = 10 * (size_t)num_dtypes;
    Staging st(Blob::STAGING, "normalise_counts");
    const uint64_t *d_counts;
    const int64_t *d_major, *d_minor;
    int64_t *d_depth;
    float *d_feats;
    st.in(&d_counts, counts, n * F);
    st.in(&d_major, major, n);
    st.in(&d_minor, minor, n);
    st.take(&d_depth, n);
    st.take(&d_feats, n * F);
    if (!st.alloc()) return st.result();
    st.check(launch_normalise(d_counts, d_major, d_minor, n, num_dtypes, mode, sym_indels, d_feats, d_depth, 0));
    st.out(feats_out, d_feats, n * F);
    if (depth_out) st.out(depth_out, d_depth, n);
    return st.result();
}

int mdk_pileup_counts(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag, const uint8_t *mapq,
                      const uint8_t *dtype, const uint32_t *cigar, const int64_t *cigar_off, const uint8_t *seq,
                      const int64_t *seq_off, int32_t start, int32_t end, int32_t num_dtypes, int32_t min_mapq,
                      int64_t max_cols, uint64_t *counts_out, int64_t *major_out, int64_t *minor_out,
                      int64_t *n_cols_out) {
    MDK_REQUIRE(n_cols_out, MDK_ERR_ARG, "pileup_counts: n_cols_out is NULL");
    *n_cols_out = 0;
    MDK_REQUIRE(n_rec >= 0 && end >= start && max_cols >= 0, MDK_ERR_ARG, "pileup_counts: bad sizes");
    MDK_REQUIRE(num_dtypes >= 1 && num_dtypes <= 4, MDK_ERR_UNSUPPORTED, "pileup_counts: 1..4 dtypes supported");
    if (n_rec == 0 || end == start) return MDK_OK;
    MDK_REQUIRE(pos && flag && mapq && dtype && cigar && cigar_off && seq && seq_off, MDK_ERR_ARG,
                "pileup_counts: NULL record array");
    MDK_REQUIRE(max_cols == 0 || (counts_out && major_out && minor_out), MDK_ERR_ARG, "pileup_counts: NULL output");
    return pileup_host("pileup_counts", device, n_rec, Records{pos, flag, mapq, dtype, cigar, cigar_off, seq, seq_off},
                       start, end, num_dtypes, min_mapq, max_cols, counts_out, nullptr, major_out, minor_out, n_cols_out);
}

// Fused featuriser: records -> counts -> normalised features without the counts ever leaving the device (SURVEY.md 8f row
// f3: "a1 -> a3 fused").  Same arguments as mdk_pileup_counts plus the normalisation switches of mdk_normalise_counts;
// copies out 64 B per column (F = 10: features 40, depth 8, positions 16) instead of 96 B out, 96 B back in and 48 B out.
int mdk_pileup_features(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag, const uint8_t *mapq,
                        const uint8_t *dtype, const uint32_t *cigar, const int64_t *cigar_off, const uint8_t *seq,
                        const int64_t *seq_off, int32_t start, int32_t end, int32_t num_dtypes, int32_t min_mapq,
                        int32_t mode, int32_t sym_indels, int64_t max_cols, float *feats_out, int64_t *depth_out,
                        int64_t *major_out, int64_t *minor_out, int64_t *n_cols_out) {
    MDK_REQUIRE(n_cols_out, MDK_ERR_ARG, "pileup_features: n_cols_out is NULL");
    *n_cols_out = 0;
    MDK_REQUIRE(n_rec >= 0 && end >= start && max_cols >= 0, MDK_ERR_ARG, "pileup_features: bad sizes");
    MDK_REQUIRE(num_dtypes >= 1 && num_dtypes <= 4, MDK_ERR_UNSUPPORTED, "pileup_features: 1..4 dtypes supported");
    MDK_REQUIRE(mode >= MDK_NORM_TOTAL && mode <= MDK_NORM_NONE, MDK_ERR_ARG, "pileup_features: unknown mode");
    if (n_rec == 0 || end == start) return MDK_OK;
    MDK_REQUIRE(pos && flag && mapq && dtype && cigar && cigar_off && seq && seq_off, MDK_ERR_ARG,
                "pileup_features: NULL record array");
    MDK_REQUIRE(max_cols == 0 || (feats_out && major_out && minor_out), MDK_ERR_ARG, "pileup_features: NULL output");
    const Normalise norm{mode, sym_indels, feats_out, depth_out};
    return pileup_host("pileup_features", device, n_rec, Records{pos, flag, mapq, dtype, cigar, cigar_off, seq, seq_off},
                       start, end, num_dtypes, min_mapq, max_cols, nullptr, &norm, major_out, minor_out, n_cols_out);
}

int mdk_read_matrix(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag, const uint8_t *mapq,
                               const uint8_t *dtype, const uint32_t *cigar, const int64_t *cigar_off, const uint8_t *seq,
                               const int64_t *seq_off, const uint8_t *qual, const int64_t *qual_off, const uint8_t *aux,
                               const int64_t *aux_off, const char *names, const int64_t *name_off, int32_t start,
                               int32_t end, int32_t num_dtypes, int32_t min_mapq, int32_t row_per_read,
                               int32_t include_dwells, int32_t include_haplotype, int32_t max_reads, int64_t max_cols,
                               int64_t max_cells, int8_t *matrix_out, int64_t *major_out, int64_t *minor_out,
                               int64_t *n_cols_out, int32_t *n_reads_out, int32_t *left_read_out,
                               int32_t *right_read_out) {
    MDK_REQUIRE(n_cols_out && n_reads_out, MDK_ERR_ARG, "read_matrix: NULL size output");
    *n_cols_out = 0;
    *n_reads_out = 0;
    MDK_REQUIRE(n_rec >= 0 && end >= start && max_cols >= 0 && max_cells >= 0 && max_reads >= 0, MDK_ERR_ARG, "read_matrix: bad sizes");
    MDK_REQUIRE(num_dtypes >= 1 && num_dtypes <= 127, MDK_ERR_UNSUPPORTED, "read_matrix: 1..127 dtypes");
    if (n_rec == 0 || end == start) return MDK_OK;
    MDK_REQUIRE(pos && flag && mapq && dtype && cigar && cigar_off && seq && seq_off && qual && qual_off && names && name_off,
                MDK_ERR_ARG, "read_matrix: NULL record array");
    MDK_REQUIRE(!(include_dwells || include_haplotype) || (aux && aux_off), MDK_ERR_ARG, "read_matrix: dwells / haplotype need the aux fields");
    const int32_t L = end - start;
    const int featlen = 4 + (include_dwells ? 1 : 0) + (include_haplotype ? 1 : 0) + (num_dtypes > 1 ? 1 : 0);
    const int f_dwell = include_dwells ? 4 : -1;
    const int f_hap = include_haplotype ? 4 + (include_dwells ? 1 : 0) : -1;
    const int f_dtype = num_dtypes > 1 ? featlen - 1 : -1;

    // ---- per read: first active position, ref_end; region depth (what bam_mplp_auto lists per position, n_plp)
    std::vector<RmHostRead> hr((size_t)n_rec);
    std::vector<int32_t> depth((size_t)L + 1, 0);
    int64_t beyond = INT64_MAX, last_cov = -1;
    for (int64_t r = 0; r < n_rec; ++r) {
        if ((flag[r] & PLP_FILTER_FLAGS) || (int)mapq[r] < min_mapq) continue;
        int64_t x = pos[r], md = 0;
        int32_t first = -1;
        for (int64_t k = cigar_off[r]; k < cigar_off[r + 1]; ++k) {
            const int op = cigar[k] & 0xF;
            const int64_t len = cigar[k] >> 4;
            if (op == OP_M || op == OP_D || op == OP_EQ || op == OP_X) {
                md += len;
                if (first < 0 && len > 0) {
                    const int64_t lo = std::max<int64_t>(x, start), hi = std::min<int64_t>(x + len, end);
                    if (lo < hi) first = (int32_t)lo;
                }
                x += len;
            } else if (op == OP_N) {
                x += len;
            }
        }
        hr[(size_t)r].first_active = first;
        hr[(size_t)r].ref_end = (int64_t)pos[r] + md;
        const int64_t lo = std::max<int64_t>(pos[r], start), hi = std::min<int64_t>(x, end);
        if (lo < hi) { depth[(size_t)(lo - start)] += 1; depth[(size_t)(hi - start)] -= 1; }
        if (x > pos[r]) {
            if (x > end) beyond = std::min<int64_t>(beyond, std::max<int64_t>(pos[r], end));
            last_cov = std::max<int64_t>(last_cov, x - 1);
        }
    }
    // `pos` when the reference's column loop ends (:337-341): the first listed position at or behind `end`, else the last
    const int64_t final_pos = beyond != INT64_MAX ? beyond : std::max<int64_t>(last_cov, 0);
    // reads bucketed by first active position (file order inside a bucket)
    std::vector<int32_t> bucket_off((size_t)L + 1, 0);
    for (int64_t r = 0; r < n_rec; ++r)
        if (hr[(size_t)r].first_active >= 0) bucket_off[(size_t)(hr[(size_t)r].first_active - start) + 1]++;
    for (int32_t i = 0; i < L; ++i) bucket_off[(size_t)i + 1] += bucket_off[(size_t)i];
    std::vector<int32_t> bucket((size_t)bucket_off[(size_t)L]);
    {
        std::vector<int32_t> fill(bucket_off.begin(), bucket_off.end() - 1);
        for (int64_t r = 0; r < n_rec; ++r)
            if (hr[(size_t)r].first_active >= 0) bucket[(size_t)fill[(size_t)(hr[(size_t)r].first_active - start)]++] = (int32_t)r;
    }
    // ---- the row bookkeeping
    std::vector<int32_t> row((size_t)n_rec, -1);
    struct Slot { int64_t ref_end; int32_t read; };
    std::vector<Slot> slots;
    std::unordered_map<std::string, int32_t> by_name;
    std::vector<int32_t> left_of;      // row -> read written at the first column
    int64_t buffer_reads = std::min<int64_t>(max_reads, 100), max_n_reads = 0;
    bool first_col = true;
    int32_t d = 0;
    const int64_t min_gap = 5;
    for (int32_t i = 0; i < L; ++i) {
        d += depth[(size_t)i];
        if (d <= 0) continue;
        const int64_t P = (int64_t)start + i, n_plp = d;
        if (n_plp > max_n_reads) max_n_reads = n_plp;
        if (buffer_reads < max_reads && max_n_reads + (row_per_read ? n_plp : 0) > buffer_reads)
            buffer_reads = std::min<int64_t>(max_reads, std::max<int64_t>(max_n_reads + (row_per_read ? n_plp : 0), 2 * buffer_reads));
        for (int32_t b = bucket_off[(size_t)i]; b < bucket_off[(size_t)i + 1]; ++b) {
            const int32_t r = bucket[(size_t)b];
            std::string nm(names + name_off[r], (size_t)(name_off[r + 1] - name_off[r]));
            int64_t read_i;
            auto it = by_name.find(nm);
            if (it != by_name.end()) {
                read_i = it->second;                   // a second alignment of a known name shares its row (:386-388)
            } else {
                const int64_t array_size = (int64_t)slots.size();
                read_i = array_size;
                if (!row_per_read) {
                    for (int64_t q = 0; q < array_size; ++q)
                        if (P >= slots[(size_t)q].ref_end + min_gap) { read_i = q; break; }
                } else if (array_size > max_n_reads) {
                    max_n_reads = array_size;
                }
                if (read_i < array_size) {
                    slots[(size_t)read_i] = Slot{hr[(size_t)r].ref_end, r};
                } else if (read_i < buffer_reads) {
                    slots.push_back(Slot{hr[(size_t)r].ref_end, r});
                }
                by_name.emplace(std::move(nm), (int32_t)read_i);
            }
            // a read that found no row stays out (the reference would let it alias a row pushed after a later growth of
            // its buffer - undefined behaviour there, not reproduced here)
            if (read_i < buffer_reads && read_i < (int64_t)slots.size()) {
                row[(size_t)r] = (int32_t)read_i;
                if (first_col) {
                    if ((int64_t)left_of.size() <= read_i) left_of.resize((size_t)read_i + 1, -1);
                    left_of[(size_t)read_i] = slots[(size_t)read_i].read;
                }
            }
        }
        first_col = false;
    }
    int64_t n_reads = row_per_read ? (int64_t)slots.size() : max_n_reads;
    n_reads = std::min<int64_t>(max_reads, n_reads);
    *n_reads_out = (int32_t)n_reads;
    // per row of the read array: the read at the first column, and the last read placed if it reaches final_pos (:559-575);
    // -1 = "__blank_k", -2 = beyond the read array (NULL id).  Handed over only with the data (the caller's arrays hold
    // n_reads entries once it knows n_reads).
    std::vector<int32_t> left_ids((size_t)n_reads, -2), right_ids((size_t)n_reads, -2);
    for (int64_t q = 0; q < n_reads && q < (int64_t)slots.size(); ++q) {
        left_ids[(size_t)q] = q < (int64_t)left_of.size() ? left_of[(size_t)q] : -1;
        right_ids[(size_t)q] = slots[(size_t)q].ref_end >= final_pos ? slots[(size_t)q].read : -1;
    }
    // ---- dwell / haplotype channels from the aux fields
    const int64_t n_ops = cigar_off[n_rec], n_qual = qual_off[n_rec];
    std::vector<int8_t> dwell;
    std::vector<uint8_t> has_dwell, hap;
    if (include_dwells) { dwell.assign((size_t)n_qual, 0); has_dwell.assign((size_t)n_rec, 0); }
    if (include_haplotype) hap.assign((size_t)n_rec, 0);
    if (include_dwells || include_haplotype) {
        for (int64_t r = 0; r < n_rec; ++r) {
            if (row[(size_t)r] < 0) continue;
            const uint8_t *mv; char mv_type; uint32_t mv_len; int hp;
            rm_scan_aux(aux + aux_off[r], aux_off[r + 1] - aux_off[r], &mv, &mv_type, &mv_len, &hp);
            if (include_haplotype) hap[(size_t)r] = (uint8_t)hp;
            if (include_dwells)
                has_dwell[(size_t)r] = rm_dwells(mv, mv_type, mv_len, (flag[r] & 0x10) != 0, (int32_t)(qual_off[r + 1] - qual_off[r]),
                                                 dwell.data() + qual_off[r]) ? 1 : 0;
        }
    }
    // ---- device: records in, columns + matrix out
    MDK_CUDA(cudaSetDevice(device));
    const int64_t cell_cap = std::min<int64_t>(max_cells, max_cols * std::max<int64_t>(n_reads, 1) * featlen);
    Staging st(Blob::STAGING, "read_matrix");
    Records recs;
    stage_records(st, n_rec, Records{pos, flag, mapq, dtype, cigar, cigar_off, seq, seq_off}, &recs);
    const uint8_t *d_qual, *d_has_dwell = nullptr, *d_hap = nullptr;
    const int64_t *d_qual_off;
    const int8_t *d_dwell = nullptr;
    const int32_t *d_row;
    int64_t *d_major, *d_minor;
    int8_t *d_matrix;
    st.in(&d_qual, qual, n_qual);
    st.in(&d_qual_off, qual_off, n_rec + 1);
    if (include_dwells) {
        st.in(&d_dwell, dwell.data(), n_qual);
        st.in(&d_has_dwell, has_dwell.data(), n_rec);
    }
    if (include_haplotype) st.in(&d_hap, hap.data(), n_rec);
    st.in(&d_row, row.data(), n_rec);
    st.take(&d_major, max_cols);
    st.take(&d_minor, max_cols);
    st.take(&d_matrix, cell_cap);
    if (!st.alloc()) return st.result();
    // the matrix is only filled when the caller's buffers hold it: columns are counted first
    const int64_t rows_dev = n_reads;
    int64_t fill_cols = max_cols;
    if (rows_dev > 0 && max_cols * rows_dev * featlen > cell_cap) fill_cols = 0;
    int rc = read_matrix_dev(n_rec, recs, n_ops, d_qual, d_qual_off, d_dwell, d_has_dwell, d_hap, d_row, start, end, min_mapq,
                             (int)rows_dev, featlen, f_dwell, f_hap, f_dtype, fill_cols, d_matrix, d_major, d_minor,
                             n_cols_out, 0);
    if (rc) return rc;
    const int64_t n_cols = *n_cols_out;
    if (n_cols > max_cols || n_cols * n_reads * featlen > max_cells || fill_cols == 0) {
        if (n_cols == 0) return MDK_OK;
        set_error("read_matrix: output buffers too small (see *n_cols_out, *n_reads_out)");
        return MDK_ERR_NOMEM;
    }
    if (n_cols > 0) {
        MDK_REQUIRE(major_out && minor_out && (matrix_out || n_reads == 0), MDK_ERR_ARG, "read_matrix: NULL output");
        st.out(major_out, d_major, n_cols);
        st.out(minor_out, d_minor, n_cols);
        st.out(matrix_out, d_matrix, n_cols * n_reads * featlen);
    }
    if (!st.ok()) return st.result();
    if (left_read_out && right_read_out && n_reads > 0) {
        memcpy(left_read_out, left_ids.data(), (size_t)n_reads * 4);
        memcpy(right_read_out, right_ids.data(), (size_t)n_reads * 4);
    }
    return MDK_OK;
}

int mdk_truth_labels(int device, int32_t pos, const uint32_t *cigar, int64_t n_cigar, const uint8_t *seq, int64_t l_seq,
                     int32_t clip_start, int32_t clip_end, int64_t n_cols, const int64_t *major, const int64_t *minor,
                     int64_t *labels_out) {
    MDK_REQUIRE(n_cigar >= 0 && l_seq >= 0 && n_cols >= 0, MDK_ERR_ARG, "truth_labels: bad sizes");
    if (n_cols == 0) return MDK_OK;
    MDK_REQUIRE(major && minor && labels_out, MDK_ERR_ARG, "truth_labels: NULL column array");
    MDK_REQUIRE((cigar || n_cigar == 0) && (seq || l_seq == 0), MDK_ERR_ARG, "truth_labels: NULL record array");
    // the kernels read the bases the CIGAR names: its query length must be the sequence's, and every base a label
    int64_t qlen = 0;
    for (int64_t k = 0; k < n_cigar; ++k)
        if (consumes_qry((int)(cigar[k] & 0xF))) qlen += cigar[k] >> 4;
    MDK_REQUIRE(qlen == l_seq, MDK_ERR_ARG, "truth_labels: CIGAR query length differs from l_seq");
    for (int64_t q = 0; q < l_seq; ++q) {
        const int code = (q & 1) ? (seq[q >> 1] & 0xF) : (seq[q >> 1] >> 4);
        MDK_REQUIRE(code == 1 || code == 2 || code == 4 || code == 8, MDK_ERR_ARG,
                    "truth_labels: truth sequence has a base other than A, C, G, T");
    }
    if (n_cigar == 0) {
        memset(labels_out, 0, (size_t)n_cols * sizeof(int64_t));
        return MDK_OK;
    }
    MDK_CUDA(cudaSetDevice(device));
    const int64_t n_blk = (n_cigar + SC_BLOCK - 1) / SC_BLOCK;
    Staging st(Blob::STAGING, "truth_labels");
    const uint32_t *d_cigar;
    const uint8_t *d_seq;
    const int64_t *d_major, *d_minor;
    int64_t *d_labels, *d_blk, *d_rstart, *d_qstart;
    uint8_t *d_match;
    st.in(&d_cigar, cigar, n_cigar);
    st.in(&d_seq, seq, (l_seq + 1) / 2);
    st.in(&d_major, major, n_cols);
    st.in(&d_minor, minor, n_cols);
    st.take(&d_labels, n_cols);
    st.take(&d_blk, 3 * (n_blk + 1));
    st.take(&d_rstart, n_cigar + 1);
    st.take(&d_qstart, n_cigar + 1);
    st.take(&d_match, n_cigar);
    if (!st.alloc()) return st.result();
    truth_sum_kernel<<<(unsigned)n_blk, SC_THREADS, 0, 0>>>(n_cigar, d_cigar, n_blk, d_blk);
    for (int k = 0; k < 3; ++k) st.check(launch_scan_blocks(d_blk + k * (n_blk + 1), n_blk, 0));
    truth_ops_kernel<<<(unsigned)n_blk, SC_THREADS, 0, 0>>>(n_cigar, d_cigar, pos, n_blk, d_blk, d_rstart, d_qstart,
                                                            d_match);
    truth_label_kernel<<<(unsigned)((n_cols + 255) / 256), 256, 0, 0>>>(
        n_cols, d_major, d_minor, d_blk + 3 * (n_blk + 1) - 1, d_rstart, d_qstart, d_match, d_seq, clip_start, clip_end,
        d_labels);
    st.check(cudaGetLastError());
    st.out(labels_out, d_labels, n_cols);
    return st.result();
}

}  // extern "C"
