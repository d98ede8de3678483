// medaka_b200: decoding the network's label probabilities on the device - consensus decode, stitching and variant
// decoding (SURVEY.md section 8 rows f1, f2) - and the variant-column rule.
//
// Consensus decode (labels.py:1053-1085): argmax label and phred quality per position.
//   decode_kernel / decode_f64_kernel   float32 / float64 probabilities (mdk_decode_consensus[_dev|_f64])
//
// Variant columns (src/medaka_rnn_variants.c:28-55, called from labels.py:869-887): variant_columns_kernel
// (mdk_variant_columns).
//
// Stitching (medaka/stitch.py:33-85): for every trimmed sample, argmax-decode the [n,5] label probabilities, compute the
// phred quality of the winning class, drop the gap calls and append the survivors to the contig.  Here the host plans the
// kept row ranges (medaka_b200/stitch.py), all ranges of a call are laid out back to back in one device array, and three
// launches produce the final FASTA/FASTQ bytes:
//   stitch_decode_kernel    row -> (ASCII base | 0 for gap, quality char); per-block survivor count
//   scan_blocks_kernel      exclusive scan of the block counts (pileup.cu; single block, <= a few 10^4 entries)
//   stitch_scatter_kernel   stable compaction: survivors move to block_base + rank-in-block; the first row of every
//                           range records where that range's output starts
// HBM-bound byte work: 20 B read per row + 2 B scratch written, 2 B scratch read + <= 2 B written.
// From the engine's decoded outputs (labels and quality bytes in device memory, mdk_stitch_labels_dev) the first launch
// is stitch_gather_kernel instead: the ranges' rows are gathered from wherever they lie (2 B read per row).
//
// Variant decoding (medaka/labels.py:889-1014 `decode_variants`, per joined sample): argmax-decode the [n,5] label
// probabilities keeping gaps, lay the draft out with '*' on insertion columns, mark the variant columns, cut them into
// runs and give every run the log-likelihood-ratio quality
//     sum_i phred(1 - p[i][pred_i]) - sum_i phred(1 - p[i][ref_i])        (labels.py:957-975, 387-401)
// summed left to right in the precision of the probabilities (float32 in production).  String building and VCF
// normalisation (Variant.trim, vcf.py:338-402) are O(#variants) and stay on the host.
//   vd_decode_kernel     column -> argmax label, mismatch flag, phred of the predicted and of the reference class
//   vd_group_kernel      the variant-column rule on the mismatch flags
//   vd_starts_kernel     run starts (variant column whose left neighbour is not) counted per block
//   scan_blocks_kernel   exclusive scan of the block counts (single block)
//   vd_runs_kernel       the k-th run start walks its run: length and the two left-to-right float32 sums
// HBM-bound byte work: 29 B read + 10 B written per column in the first kernel, ~12 B per column in the others.
// From the engine's variant-decoded outputs (call bytes and the two phreds in device memory, phred.cuh):
//   vd_join_cuts_kernel  per trimmed piece, the last insertion-free column whose call equals the draft - all that
//                        join_samples (medaka/variant.py:30-119) reads of the labels (mdk_variant_join_cuts)
//   vd_gather_kernel     the joined samples' pieces, from wherever they lie, into the columns vd_decode_kernel would
//                        have written, one padding column (no mismatch, not an insertion) after every joined sample so
//                        that neither the variant-column rule nor a run crosses into the next; then vd_group, vd_starts,
//                        scan_blocks and vd_runs as above, and vd_run_cols_kernel compacts the run columns' labels (and
//                        phreds) for the host (mdk_decode_variants_dev).  9 B read per column instead of 20 + 9.
#include "common.cuh"
#include "phred.cuh"

#include <vector>

namespace mdk {

namespace {

// src/medaka_rnn_variants.c:28-55: a major column is variant when it mismatches; the minor (insertion) columns that
// follow it are variant when ANY column of the group - the major or one of its minors - mismatches.  The first column is
// taken as a major ("assume start on major").  The reference walks the columns sequentially; here every column finds its
// group (insertion runs are short) and reduces over it.  mism(j): whether column j mismatches.
template <class Mism>
__device__ __forceinline__ bool variant_column(const int64_t *__restrict__ minor, int64_t n, int64_t i, Mism mism) {
    bool any = mism(i);
    if (i != 0 && minor[i] != 0) {
        for (int64_t j = i - 1; j >= 0 && !any; --j) {      // back to (and including) the group's major column
            any = mism(j);
            if (j == 0 || minor[j] == 0) break;
        }
        for (int64_t j = i + 1; j < n && !any && minor[j] != 0; ++j) any = mism(j);
    }
    return any;
}

// ---------------------------------------------------------------------------------------- consensus decode: 41 B per position
__global__ void __launch_bounds__(256) decode_kernel(const float *__restrict__ probs, int64_t n,
                                                     uint8_t *__restrict__ labels, uint8_t *__restrict__ quals) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *p = probs + i * NCLS;
    float best = p[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c) {
        const float v = p[c];
        if (v > best) { best = v; arg = c; }   // strict '>' : first maximum wins, as np.argmax
    }
    labels[i] = (uint8_t)arg;
    if (quals) quals[i] = phred_char(best);
}

// float64 probabilities (what numpy computes when label_probs is a float64 array, e.g. the reference's own
// test literals medaka/test/test_labels.py:252-266): every step in double, like numpy would.
__global__ void __launch_bounds__(256) decode_f64_kernel(const double *__restrict__ probs, int64_t n,
                                                         uint8_t *__restrict__ labels, uint8_t *__restrict__ quals) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double *p = probs + i * NCLS;
    double best = p[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c) {
        const double v = p[c];
        if (v > best) { best = v; arg = c; }
    }
    labels[i] = (uint8_t)arg;
    if (quals) {
        double err = 1.0 - best;
        err = fmin(fmax(err, 1e-7), 1.0);
        double q = -10.0 * log10(err);
        q = fmin(q, 70.0);
        quals[i] = (uint8_t)((int)q + 33);
    }
}

cudaError_t launch_decode(const float *probs, int64_t n, uint8_t *labels, uint8_t *quals, cudaStream_t s) {
    decode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(probs, n, labels, quals);
    return cudaGetLastError();
}

cudaError_t launch_decode(const double *probs, int64_t n, uint8_t *labels, uint8_t *quals, cudaStream_t s) {
    decode_f64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(probs, n, labels, quals);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------- variant columns: ~10 B per column
__global__ void __launch_bounds__(256) variant_columns_kernel(const int64_t *__restrict__ minor,
                                                              const uint8_t *__restrict__ ref,
                                                              const uint8_t *__restrict__ pred, int64_t n,
                                                              uint8_t *__restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = variant_column(minor, n, i, [&](int64_t j) { return ref[j] != pred[j]; });
}

// ---------------------------------------------------------------------------------------- stitching
constexpr int ST_THREADS = 256;
constexpr int ST_ROWS_PER_THREAD = 4;
constexpr int ST_BLOCK_ROWS = ST_THREADS * ST_ROWS_PER_THREAD;   // 1024 rows per block

// '*ACGT' (labels.py:342); 0 marks a gap call so the byte doubles as the keep flag
__device__ __forceinline__ uint8_t label_symbol(int label) {
    return (uint8_t)((0x5447434100ull >> (8 * label)) & 0xff);
}

__device__ __forceinline__ void decode_row(const float *__restrict__ p, uint8_t &sym, uint8_t &qual) {
    float best = p[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c) {
        const float v = p[c];
        if (v > best) { best = v; arg = c; }                  // first maximum wins (np.argmax)
    }
    qual = phred_char(best);
    sym = label_symbol(arg);
}

// Gather for mdk_stitch_labels_dev: concatenated row r of the call lies in segment k (seg_base[k] <= r < seg_base[k+1])
// at arena row seg_start[k] + r - seg_base[k].  Writes what stitch_decode_kernel writes (symbol | 0, quality, per-block
// survivor count), so that stitch_scatter_kernel compacts either.  Thread t owns rows [base + 4t, base + 4t + 4).
__global__ void __launch_bounds__(ST_THREADS) stitch_gather_kernel(const uint8_t *__restrict__ labels,
                                                                   const uint8_t *__restrict__ quals,
                                                                   const int64_t *__restrict__ seg_start,
                                                                   const int64_t *__restrict__ seg_base, int64_t n_seg,
                                                                   int64_t n, uint8_t *__restrict__ sym,
                                                                   uint8_t *__restrict__ qual,
                                                                   int64_t *__restrict__ block_count) {
    __shared__ uint32_t warp_cnt[ST_THREADS / 32];
    const int64_t r0 = (int64_t)blockIdx.x * ST_BLOCK_ROWS + (int64_t)threadIdx.x * ST_ROWS_PER_THREAD;
    uint32_t kept = 0;
    if (r0 < n) {
        int64_t lo = 0, hi = n_seg;     // last segment starting at or before r0
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (seg_base[mid] <= r0) lo = mid; else hi = mid;
        }
        int64_t k = lo;
        for (int j = 0; j < ST_ROWS_PER_THREAD && r0 + j < n; ++j) {
            const int64_t r = r0 + j;
            while (k + 1 < n_seg && seg_base[k + 1] <= r) ++k;
            const int64_t a = seg_start[k] + (r - seg_base[k]);
            const uint8_t l = labels[a];
            const uint8_t s = l < NCLS ? label_symbol(l) : 0;
            sym[r] = s;
            qual[r] = quals ? quals[a] : 0;
            kept += (s != 0);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = kept;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
#pragma unroll
        for (int w = 0; w < ST_THREADS / 32; ++w) t += warp_cnt[w];
        block_count[blockIdx.x] = t;
    }
}

// Thread t of a block owns rows [base + 4t, base + 4t + 4): the four outputs are one 32-bit store.
__global__ void __launch_bounds__(ST_THREADS) stitch_decode_kernel(const float *__restrict__ probs, int64_t n,
                                                                   uint8_t *__restrict__ sym,
                                                                   uint8_t *__restrict__ qual,
                                                                   int64_t *__restrict__ block_count) {
    __shared__ uint32_t warp_cnt[ST_THREADS / 32];
    const int64_t r0 = (int64_t)blockIdx.x * ST_BLOCK_ROWS + (int64_t)threadIdx.x * ST_ROWS_PER_THREAD;
    uint32_t s4 = 0, q4 = 0, kept = 0;
    if (r0 + ST_ROWS_PER_THREAD <= n) {
        // 4 rows = 20 floats = 80 B, 16-byte aligned because r0 is a multiple of 4
        const float4 *v = reinterpret_cast<const float4 *>(probs + r0 * NCLS);
        float f[20];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const float4 x = __ldcs(v + i);
            f[4 * i] = x.x; f[4 * i + 1] = x.y; f[4 * i + 2] = x.z; f[4 * i + 3] = x.w;
        }
#pragma unroll
        for (int j = 0; j < ST_ROWS_PER_THREAD; ++j) {
            uint8_t s, q;
            decode_row(f + j * NCLS, s, q);
            s4 |= (uint32_t)s << (8 * j);
            q4 |= (uint32_t)q << (8 * j);
            kept += (s != 0);
        }
        *reinterpret_cast<uint32_t *>(sym + r0) = s4;
        *reinterpret_cast<uint32_t *>(qual + r0) = q4;
    } else {
        for (int j = 0; j < ST_ROWS_PER_THREAD && r0 + j < n; ++j) {
            uint8_t s, q;
            decode_row(probs + (r0 + j) * NCLS, s, q);
            sym[r0 + j] = s;
            qual[r0 + j] = q;
            kept += (s != 0);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = kept;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
#pragma unroll
        for (int w = 0; w < ST_THREADS / 32; ++w) t += warp_cnt[w];
        block_count[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(ST_THREADS) stitch_scatter_kernel(const uint8_t *__restrict__ sym,
                                                                    const uint8_t *__restrict__ qual, int64_t n,
                                                                    const int64_t *__restrict__ block_base,
                                                                    const int64_t *__restrict__ seg_base,
                                                                    int64_t n_seg, uint8_t *__restrict__ seq_out,
                                                                    uint8_t *__restrict__ qual_out,
                                                                    int64_t *__restrict__ seg_out_off) {
    __shared__ uint32_t warp_cnt[ST_THREADS / 32];
    const int64_t r0 = (int64_t)blockIdx.x * ST_BLOCK_ROWS + (int64_t)threadIdx.x * ST_ROWS_PER_THREAD;
    uint32_t s4 = 0, q4 = 0;
    if (r0 + ST_ROWS_PER_THREAD <= n) {
        s4 = *reinterpret_cast<const uint32_t *>(sym + r0);
        q4 = *reinterpret_cast<const uint32_t *>(qual + r0);
    } else {
        for (int j = 0; j < ST_ROWS_PER_THREAD && r0 + j < n; ++j) {
            s4 |= (uint32_t)sym[r0 + j] << (8 * j);
            q4 |= (uint32_t)qual[r0 + j] << (8 * j);
        }
    }
    uint32_t mine = 0;
#pragma unroll
    for (int j = 0; j < ST_ROWS_PER_THREAD; ++j) mine += ((s4 >> (8 * j)) & 0xff) != 0;
    // exclusive rank of this thread's first survivor inside the block
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_cnt[warp] = x;
    __syncthreads();
    uint32_t before = x - mine;
    for (int w = 0; w < warp; ++w) before += warp_cnt[w];
    int64_t o = block_base[blockIdx.x] + before;
    const int64_t o_first = o;
#pragma unroll
    for (int j = 0; j < ST_ROWS_PER_THREAD; ++j) {
        const uint8_t s = (s4 >> (8 * j)) & 0xff;
        if (s) {
            seq_out[o] = s;
            if (qual_out) qual_out[o] = (q4 >> (8 * j)) & 0xff;
            ++o;
        }
    }
    // range starts: the ranges are sorted and non-empty, so the ones beginning inside this thread's four rows are a
    // contiguous slice of seg_base found by one lower_bound
    if (r0 < n) {
        int64_t lo = 0, hi = n_seg;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (seg_base[mid] < r0) lo = mid + 1; else hi = mid;
        }
        for (int64_t k = lo; k < n_seg && seg_base[k] < r0 + ST_ROWS_PER_THREAD; ++k) {
            const int j_start = (int)(seg_base[k] - r0);
            int64_t off = o_first;
            for (int j = 0; j < j_start; ++j) off += ((s4 >> (8 * j)) & 0xff) != 0;
            seg_out_off[k] = off;
        }
    }
}

// ---------------------------------------------------------------------------------------- variant decoding
constexpr int VD_THREADS = 256;

// ref_code: 0..4 = '*ACGT' (labels.py:342); 5 = 'N' (compared as a symbol of its own, scored as '*': labels.py:949-952);
// >= 6 = any other draft symbol (never equal to a call; scored as '*' - the host refuses it unless the run is skipped)
__global__ void __launch_bounds__(VD_THREADS) vd_decode_kernel(const float *__restrict__ probs,
                                                               const uint8_t *__restrict__ ref_code, int64_t n,
                                                               uint8_t *__restrict__ pred, uint8_t *__restrict__ mism,
                                                               float *__restrict__ pred_q, float *__restrict__ ref_q) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float p[NCLS];
#pragma unroll
    for (int c = 0; c < NCLS; ++c) p[c] = __ldcs(probs + i * NCLS + c);
    float best = p[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < NCLS; ++c)
        if (p[c] > best) { best = p[c]; arg = c; }          // first maximum wins (np.argmax, labels.py:1063)
    const int r = ref_code[i];
    const int rq = r < NCLS ? r : 0;
    float pr = p[0];
#pragma unroll
    for (int c = 1; c < NCLS; ++c) pr = (rq == c) ? p[c] : pr;
    pred[i] = (uint8_t)arg;
    mism[i] = (uint8_t)(r != arg);
    pred_q[i] = phred_f32(best);
    ref_q[i] = phred_f32(pr);
}

__global__ void __launch_bounds__(VD_THREADS) vd_group_kernel(const int64_t *__restrict__ minor,
                                                              const uint8_t *__restrict__ mism, int64_t n,
                                                              uint8_t *__restrict__ is_var) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    is_var[i] = variant_column(minor, n, i, [&](int64_t j) { return mism[j] != 0; });
}

__global__ void __launch_bounds__(VD_THREADS) vd_starts_kernel(const uint8_t *__restrict__ is_var, int64_t n,
                                                               int64_t *__restrict__ block_count) {
    __shared__ uint32_t warp_cnt[VD_THREADS / 32];
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    uint32_t start = 0;
    if (i < n) start = is_var[i] && (i == 0 || !is_var[i - 1]);
    const uint32_t ballot = __ballot_sync(0xffffffffu, start);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = __popc(ballot);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
#pragma unroll
        for (int w = 0; w < VD_THREADS / 32; ++w) t += warp_cnt[w];
        block_count[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(VD_THREADS) vd_runs_kernel(const uint8_t *__restrict__ is_var,
                                                             const float *__restrict__ pred_q,
                                                             const float *__restrict__ ref_q, int64_t n,
                                                             const int64_t *__restrict__ block_base, int64_t max_runs,
                                                             int64_t *__restrict__ run_start, int64_t *__restrict__ run_len,
                                                             float *__restrict__ run_pred_q, float *__restrict__ run_ref_q) {
    __shared__ uint32_t warp_cnt[VD_THREADS / 32];
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    uint32_t start = 0;
    if (i < n) start = is_var[i] && (i == 0 || !is_var[i - 1]);
    const uint32_t ballot = __ballot_sync(0xffffffffu, start);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_cnt[warp] = __popc(ballot);
    __syncthreads();
    if (!start) return;
    uint32_t before = __popc(ballot & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) before += warp_cnt[w];
    const int64_t k = block_base[blockIdx.x] + before;
    if (k >= max_runs) return;
    // Python's sum(): start from int 0, add left to right - float32 + float32 in float32
    float sp = 0.0f, sr = 0.0f;
    int64_t j = i;
    for (; j < n && is_var[j]; ++j) {
        sp += pred_q[j];
        sr += ref_q[j];
    }
    run_start[k] = i;
    run_len[k] = j - i;
    run_pred_q[k] = sp;
    run_ref_q[k] = sr;
}

// One block per piece k (rows [0, seg_rows[k]) at seg_calls[k]): cut[k] = the last column that is no insertion and whose
// call equals the draft, or -1 when every column is "different" in join_samples' sense (call != draft, or both are
// '*'; insertion columns always are), i.e. when no column has call == draft != '*'.
__global__ void __launch_bounds__(VD_THREADS) vd_join_cuts_kernel(const uint8_t *const *__restrict__ seg_calls,
                                                                  const int64_t *__restrict__ seg_rows,
                                                                  int64_t *__restrict__ cut) {
    __shared__ int64_t s_last[VD_THREADS / 32];
    __shared__ int s_any[VD_THREADS / 32];
    const uint8_t *c = seg_calls[blockIdx.x];
    const int64_t n = seg_rows[blockIdx.x];
    int64_t last = -1;
    int any = 0;
    for (int64_t i = threadIdx.x; i < n; i += VD_THREADS) {
        const uint8_t v = c[i];
        if (!(v & (VCALL_MISM | VCALL_INS))) {
            last = i;                                   // rows grow with i: the thread's last match is its largest
            any |= (v & VCALL_LABEL) != 0;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        last = max(last, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)last, o));
        any |= __shfl_xor_sync(0xffffffffu, any, o);
    }
    if ((threadIdx.x & 31) == 0) { s_last[threadIdx.x >> 5] = last; s_any[threadIdx.x >> 5] = any; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < VD_THREADS / 32; ++w) { last = max(last, s_last[w]); any |= s_any[w]; }
        cut[blockIdx.x] = any ? last : -1;
    }
}

// Padded column r of the call: segment k (the last with pstart[k] <= r) holds rows [pstart[k], pstart[k] + seg_rows[k]);
// the column just past a joined sample's last segment is its padding column.  Writes what vd_decode_kernel writes, and
// the insertion flag as vd_group_kernel's minor.  bad: set when a joined sample starts on an insertion column.
__global__ void __launch_bounds__(VD_THREADS) vd_gather_kernel(const uint8_t *const *__restrict__ seg_calls,
                                                               const float *const *__restrict__ seg_pq,
                                                               const float *__restrict__ const *seg_rq,
                                                               const int64_t *__restrict__ pstart,
                                                               const int64_t *__restrict__ seg_rows,
                                                               const uint8_t *__restrict__ seg_first, int64_t n_seg,
                                                               int64_t n, uint8_t *__restrict__ pred,
                                                               uint8_t *__restrict__ mism, int64_t *__restrict__ minor,
                                                               float *__restrict__ pred_q, float *__restrict__ ref_q,
                                                               int *__restrict__ bad) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    int64_t lo = 0, hi = n_seg;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (pstart[mid] <= r) lo = mid; else hi = mid;
    }
    const int64_t j = r - pstart[lo];
    if (j >= seg_rows[lo]) {                                      // padding
        pred[r] = 0; mism[r] = 0; minor[r] = 0; pred_q[r] = 0.f; ref_q[r] = 0.f;
        return;
    }
    const uint8_t v = seg_calls[lo][j];
    pred[r] = v & VCALL_LABEL;
    mism[r] = (v & VCALL_MISM) != 0;
    minor[r] = (v & VCALL_INS) != 0;
    pred_q[r] = seg_pq[lo][j];
    ref_q[r] = seg_rq[lo][j];
    if (j == 0 && seg_first[lo] && (v & VCALL_INS)) atomicOr(bad, 1);
}

// Run k's columns [run_start[k], run_start[k] + run_len[k]) to [off[k], off[k] + run_len[k]) of the compact outputs
__global__ void __launch_bounds__(VD_THREADS) vd_run_cols_kernel(const uint8_t *__restrict__ pred,
                                                                 const float *__restrict__ pred_q,
                                                                 const float *__restrict__ ref_q,
                                                                 const int64_t *__restrict__ run_start,
                                                                 const int64_t *__restrict__ run_len,
                                                                 const int64_t *__restrict__ off, int64_t n_runs,
                                                                 uint8_t *__restrict__ cols_pred,
                                                                 float *__restrict__ cols_pq, float *__restrict__ cols_rq) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_runs) return;
    const int64_t a = run_start[k], o = off[k];
    for (int64_t j = 0; j < run_len[k]; ++j) {
        cols_pred[o + j] = pred[a + j];
        if (cols_pq) { cols_pq[o + j] = pred_q[a + j]; cols_rq[o + j] = ref_q[a + j]; }
    }
}

// mdk_decode_consensus and mdk_decode_consensus_f64: the same staging for either probability type
template <class P>
int decode_host(const char *what, int device, const P *probs, int64_t n, uint8_t *labels_out, uint8_t *quals_out) {
    MDK_REQUIRE(n >= 0, MDK_ERR_ARG, "decode_consensus: n < 0");
    if (n == 0) return MDK_OK;
    MDK_REQUIRE(probs && labels_out, MDK_ERR_ARG, "decode_consensus: NULL pointer");
    MDK_CUDA(cudaSetDevice(device));
    Staging st(Blob::STAGING, what);
    const P *d_probs;
    uint8_t *d_labels, *d_quals;
    st.in(&d_probs, probs, n * NCLS);
    st.take(&d_labels, n);
    st.take(&d_quals, n);
    if (!st.alloc()) return st.result();
    st.check(launch_decode(d_probs, n, d_labels, quals_out ? d_quals : nullptr, 0));
    st.out(labels_out, d_labels, n);
    if (quals_out) st.out(quals_out, d_quals, n);
    return st.result();
}

}  // namespace

}  // namespace mdk

using namespace mdk;

extern "C" {

int mdk_decode_consensus_dev(int device, const float *probs_dev, int64_t n, uint8_t *labels_out_dev,
                             uint8_t *quals_out_dev) {
    MDK_REQUIRE(n >= 0, MDK_ERR_ARG, "decode_consensus: n < 0");
    if (n == 0) return MDK_OK;
    MDK_REQUIRE(probs_dev && labels_out_dev, MDK_ERR_ARG, "decode_consensus: NULL pointer");
    MDK_CUDA(cudaSetDevice(device));
    MDK_CUDA(launch_decode(probs_dev, n, labels_out_dev, quals_out_dev, 0));
    return MDK_OK;
}

int mdk_decode_consensus(int device, const float *probs, int64_t n, uint8_t *labels_out, uint8_t *quals_out) {
    return decode_host("decode_consensus", device, probs, n, labels_out, quals_out);
}

int mdk_decode_consensus_f64(int device, const double *probs, int64_t n, uint8_t *labels_out, uint8_t *quals_out) {
    return decode_host("decode_consensus_f64", device, probs, n, labels_out, quals_out);
}

int mdk_variant_columns(int device, const int64_t *minor, const uint8_t *reference, const uint8_t *prediction,
                        uint8_t *out, int64_t len) {
    MDK_REQUIRE(len >= 0, MDK_ERR_ARG, "variant_columns: len < 0");
    if (len == 0) return MDK_OK;
    MDK_REQUIRE(minor && reference && prediction && out, MDK_ERR_ARG, "variant_columns: NULL pointer");
    MDK_CUDA(cudaSetDevice(device));
    Staging st(Blob::STAGING, "variant_columns");
    const int64_t *d_minor;
    const uint8_t *d_ref, *d_pred;
    uint8_t *d_out;
    st.in(&d_minor, minor, len);
    st.in(&d_ref, reference, len);
    st.in(&d_pred, prediction, len);
    st.take(&d_out, len);
    if (!st.alloc()) return st.result();
    variant_columns_kernel<<<(unsigned)((len + 255) / 256), 256, 0, 0>>>(d_minor, d_ref, d_pred, len, d_out);
    st.check(cudaGetLastError());
    st.out(out, d_out, len);
    return st.result();
}

// The ranges' rows are decoded, the survivors compacted into seq_out_dev / qual_out_dev; the staging of seg_base and
// the kernels' scratch share the SCRATCH blob (mdk_stitch_consensus holds the STAGING one).
int mdk_stitch_consensus_dev(int device, const float *probs_dev, int64_t n_rows, const int64_t *seg_base,
                             int64_t n_seg, uint8_t *seq_out_dev, uint8_t *qual_out_dev, int64_t *seg_out_off) {
    MDK_REQUIRE(n_rows >= 0 && n_seg >= 0, MDK_ERR_ARG, "stitch_consensus: negative size");
    MDK_REQUIRE(seg_out_off, MDK_ERR_ARG, "stitch_consensus: NULL seg_out_off");
    if (n_rows == 0 || n_seg == 0) {
        MDK_REQUIRE(n_rows == 0 && n_seg == 0, MDK_ERR_ARG, "stitch_consensus: rows without ranges (or vice versa)");
        seg_out_off[0] = 0;
        return MDK_OK;
    }
    MDK_REQUIRE(probs_dev && seg_base && seq_out_dev, MDK_ERR_ARG, "stitch_consensus: NULL pointer");
    MDK_REQUIRE(seg_base[0] == 0, MDK_ERR_ARG, "stitch_consensus: first range must start at row 0");
    for (int64_t k = 1; k < n_seg; ++k)
        MDK_REQUIRE(seg_base[k] > seg_base[k - 1] && seg_base[k] < n_rows, MDK_ERR_ARG,
                    "stitch_consensus: range starts must be strictly increasing and < n_rows");
    MDK_CUDA(cudaSetDevice(device));
    const int64_t n_blocks = (n_rows + ST_BLOCK_ROWS - 1) / ST_BLOCK_ROWS;
    const int64_t n4 = (n_rows + 3) & ~(int64_t)3;      // whole 32-bit stores of four rows
    Staging st(Blob::SCRATCH, "stitch_consensus_dev");
    const int64_t *d_seg;
    int64_t *d_off, *d_base;
    uint8_t *d_sym, *d_qual;
    st.in(&d_seg, seg_base, n_seg);
    st.take(&d_off, n_seg + 1);
    st.take(&d_sym, n4);
    st.take(&d_qual, n4);
    st.take(&d_base, n_blocks + 1);
    if (!st.alloc()) return st.result();
    stitch_decode_kernel<<<(unsigned)n_blocks, ST_THREADS, 0, 0>>>(probs_dev, n_rows, d_sym, d_qual, d_base);
    st.check(launch_scan_blocks(d_base, n_blocks, 0));
    stitch_scatter_kernel<<<(unsigned)n_blocks, ST_THREADS, 0, 0>>>(d_sym, d_qual, n_rows, d_base, d_seg, n_seg,
                                                                    seq_out_dev, qual_out_dev, d_off);
    st.check(cudaGetLastError());
    // total survivors -> seg_out_off[n_seg]
    if (st.ok()) st.check(cudaMemcpyAsync(d_off + n_seg, d_base + n_blocks, sizeof(int64_t), cudaMemcpyDeviceToDevice, 0));
    st.out(seg_out_off, d_off, n_seg + 1);
    return st.result();
}

int mdk_stitch_consensus(int device, const float *const *seg_probs, const int64_t *seg_rows, int64_t n_seg,
                         uint8_t *seq_out, uint8_t *qual_out, int64_t *seg_out_off) {
    MDK_REQUIRE(n_seg >= 0, MDK_ERR_ARG, "stitch_consensus: n_seg < 0");
    MDK_REQUIRE(seg_out_off, MDK_ERR_ARG, "stitch_consensus: NULL seg_out_off");
    if (n_seg == 0) { seg_out_off[0] = 0; return MDK_OK; }
    MDK_REQUIRE(seg_probs && seg_rows && seq_out, MDK_ERR_ARG, "stitch_consensus: NULL pointer");
    int64_t n = 0;
    std::vector<int64_t> base((size_t)n_seg);
    for (int64_t k = 0; k < n_seg; ++k) {
        MDK_REQUIRE(seg_rows[k] > 0 && seg_probs[k], MDK_ERR_ARG,
                    "stitch_consensus: every range needs rows > 0 and a probabilities pointer");
        base[(size_t)k] = n;
        n += seg_rows[k];
    }
    MDK_CUDA(cudaSetDevice(device));
    Staging st(Blob::STAGING, "stitch_consensus");
    float *d_probs;
    uint8_t *d_seq, *d_qual;
    st.take(&d_probs, (size_t)n * NCLS);
    st.take(&d_seq, n);
    st.take(&d_qual, n);
    if (!st.alloc()) return st.result();
    for (int64_t k = 0; k < n_seg; ++k)      // the ranges back to back
        if (st.ok()) st.check(cudaMemcpyAsync(d_probs + base[(size_t)k] * NCLS, seg_probs[k], (size_t)seg_rows[k] * NCLS * 4,
                                              cudaMemcpyHostToDevice, 0));
    if (!st.ok()) return st.result();
    int rc = mdk_stitch_consensus_dev(device, d_probs, n, base.data(), n_seg, d_seq, qual_out ? d_qual : nullptr,
                                      seg_out_off);
    if (rc) return rc;
    st.out(seq_out, d_seq, seg_out_off[n_seg]);
    if (qual_out) st.out(qual_out, d_qual, seg_out_off[n_seg]);
    return st.result();
}

// Segments are row ranges of the engine's decoded outputs (mdk_engine_submit_decoded) anywhere in device memory; they are
// concatenated in call order, gathered into the stitch scratch and compacted by the kernels mdk_stitch_consensus runs.
int mdk_stitch_labels_dev(int device, const uint8_t *labels_dev, const uint8_t *quals_dev, const int64_t *seg_start,
                          const int64_t *seg_rows, int64_t n_seg, uint8_t *seq_out, uint8_t *qual_out,
                          int64_t *seg_out_off) {
    MDK_REQUIRE(n_seg >= 0, MDK_ERR_ARG, "stitch_labels: n_seg < 0");
    MDK_REQUIRE(seg_out_off, MDK_ERR_ARG, "stitch_labels: NULL seg_out_off");
    if (n_seg == 0) { seg_out_off[0] = 0; return MDK_OK; }
    MDK_REQUIRE(labels_dev && seg_start && seg_rows && seq_out, MDK_ERR_ARG, "stitch_labels: NULL pointer");
    std::vector<int64_t> base((size_t)n_seg);
    int64_t n = 0;
    for (int64_t k = 0; k < n_seg; ++k) {
        MDK_REQUIRE(seg_rows[k] > 0, MDK_ERR_ARG, "stitch_labels: every segment needs rows > 0");
        base[(size_t)k] = n;
        n += seg_rows[k];
    }
    MDK_CUDA(cudaSetDevice(device));
    const int64_t n_blocks = (n + ST_BLOCK_ROWS - 1) / ST_BLOCK_ROWS;
    const int64_t n4 = (n + 3) & ~(int64_t)3;      // whole 32-bit loads of four rows in the scatter
    Staging st(Blob::STAGING, "stitch_labels_dev");
    const int64_t *d_start, *d_seg;
    int64_t *d_off, *d_base;
    uint8_t *d_sym, *d_qual, *d_seq, *d_qout = nullptr;
    st.in(&d_start, seg_start, n_seg);
    st.in(&d_seg, base.data(), n_seg);
    st.take(&d_off, n_seg + 1);
    st.take(&d_base, n_blocks + 1);
    st.take(&d_sym, n4);
    st.take(&d_qual, n4);
    st.take(&d_seq, n);
    if (qual_out) st.take(&d_qout, n);
    if (!st.alloc()) return st.result();
    stitch_gather_kernel<<<(unsigned)n_blocks, ST_THREADS, 0, 0>>>(labels_dev, quals_dev, d_start, d_seg, n_seg, n,
                                                                   d_sym, d_qual, d_base);
    st.check(cudaGetLastError());
    st.check(launch_scan_blocks(d_base, n_blocks, 0));
    stitch_scatter_kernel<<<(unsigned)n_blocks, ST_THREADS, 0, 0>>>(d_sym, d_qual, n, d_base, d_seg, n_seg, d_seq,
                                                                    d_qout, d_off);
    st.check(cudaGetLastError());
    if (st.ok()) st.check(cudaMemcpyAsync(d_off + n_seg, d_base + n_blocks, sizeof(int64_t), cudaMemcpyDeviceToDevice, 0));
    st.out(seg_out_off, d_off, n_seg + 1);
    if (!st.ok()) return st.result();
    st.out(seq_out, d_seq, seg_out_off[n_seg]);
    if (qual_out) st.out(qual_out, d_qout, seg_out_off[n_seg]);
    return st.result();
}

int mdk_decode_variants(int device, const float *probs, const int64_t *minor, const uint8_t *ref_code, int64_t n,
                        uint8_t *pred_out, uint8_t *is_var_out, float *pred_q_out, float *ref_q_out, int64_t max_runs,
                        int64_t *run_start, int64_t *run_len, float *run_pred_q, float *run_ref_q,
                        int64_t *n_runs_out) {
    MDK_REQUIRE(n_runs_out, MDK_ERR_ARG, "decode_variants: n_runs_out is NULL");
    *n_runs_out = 0;
    MDK_REQUIRE(n >= 0 && max_runs >= 0, MDK_ERR_ARG, "decode_variants: negative size");
    if (n == 0) return MDK_OK;
    MDK_REQUIRE(probs && minor && ref_code && pred_out && is_var_out, MDK_ERR_ARG, "decode_variants: NULL pointer");
    MDK_REQUIRE(max_runs == 0 || (run_start && run_len && run_pred_q && run_ref_q), MDK_ERR_ARG,
                "decode_variants: NULL run output");
    MDK_REQUIRE(minor[0] == 0, MDK_ERR_ARG,
                "decode_variants: the first position of a sample must not be an insertion (labels.py:909-911)");
    MDK_CUDA(cudaSetDevice(device));
    const int64_t n_blocks = (n + VD_THREADS - 1) / VD_THREADS;
    Staging st(Blob::STAGING, "decode_variants");
    const float *d_probs;
    const int64_t *d_minor;
    const uint8_t *d_ref;
    uint8_t *d_pred, *d_mism, *d_var;
    float *d_pq, *d_rq, *d_rp, *d_rr;
    int64_t *d_base, *d_rs, *d_rl;
    st.in(&d_probs, probs, n * NCLS);
    st.in(&d_minor, minor, n);
    st.in(&d_ref, ref_code, n);
    st.take(&d_pred, n);
    st.take(&d_mism, n);
    st.take(&d_var, n);
    st.take(&d_pq, n);
    st.take(&d_rq, n);
    st.take(&d_base, n_blocks + 1);
    st.take(&d_rs, max_runs);
    st.take(&d_rl, max_runs);
    st.take(&d_rp, max_runs);
    st.take(&d_rr, max_runs);
    if (!st.alloc()) return st.result();
    const unsigned g = (unsigned)n_blocks;
    vd_decode_kernel<<<g, VD_THREADS, 0, 0>>>(d_probs, d_ref, n, d_pred, d_mism, d_pq, d_rq);
    vd_group_kernel<<<g, VD_THREADS, 0, 0>>>(d_minor, d_mism, n, d_var);
    vd_starts_kernel<<<g, VD_THREADS, 0, 0>>>(d_var, n, d_base);
    st.check(launch_scan_blocks(d_base, n_blocks, 0));
    vd_runs_kernel<<<g, VD_THREADS, 0, 0>>>(d_var, d_pq, d_rq, n, d_base, max_runs, d_rs, d_rl, d_rp, d_rr);
    st.check(cudaGetLastError());
    int64_t total = 0;
    st.out(&total, d_base + n_blocks, 1);
    st.out(pred_out, d_pred, n);
    st.out(is_var_out, d_var, n);
    if (pred_q_out) st.out(pred_q_out, d_pq, n);
    if (ref_q_out) st.out(ref_q_out, d_rq, n);
    if (!st.ok()) return st.result();
    *n_runs_out = total;
    if (total > max_runs) {
        set_error("decode_variants: run buffers too small (see *n_runs_out)");
        return MDK_ERR_NOMEM;
    }
    st.out(run_start, d_rs, total);
    st.out(run_len, d_rl, total);
    st.out(run_pred_q, d_rp, total);
    st.out(run_ref_q, d_rr, total);
    return st.result();
}

// Pieces are row ranges of the engine's variant-decoded outputs anywhere in device memory; one block per piece.
int mdk_variant_join_cuts(int device, const uint8_t *const *seg_calls, const int64_t *seg_rows, int64_t n_seg,
                          int64_t *cut_out) {
    MDK_REQUIRE(n_seg >= 0, MDK_ERR_ARG, "variant_join_cuts: n_seg < 0");
    if (n_seg == 0) return MDK_OK;
    MDK_REQUIRE(seg_calls && seg_rows && cut_out, MDK_ERR_ARG, "variant_join_cuts: NULL pointer");
    MDK_REQUIRE(n_seg < ((int64_t)1 << 31), MDK_ERR_ARG, "variant_join_cuts: too many pieces");
    for (int64_t k = 0; k < n_seg; ++k)
        MDK_REQUIRE(seg_rows[k] > 0 && seg_calls[k], MDK_ERR_ARG, "variant_join_cuts: every piece needs rows > 0");
    MDK_CUDA(cudaSetDevice(device));
    Staging st(Blob::STAGING, "variant_join_cuts");
    const uint8_t *const *d_calls;
    const int64_t *d_rows;
    int64_t *d_cut;
    st.in(&d_calls, seg_calls, n_seg);
    st.in(&d_rows, seg_rows, n_seg);
    st.take(&d_cut, n_seg);
    if (!st.alloc()) return st.result();
    vd_join_cuts_kernel<<<(unsigned)n_seg, VD_THREADS, 0, 0>>>(d_calls, d_rows, d_cut);
    st.check(cudaGetLastError());
    st.out(cut_out, d_cut, n_seg);
    return st.result();
}

// The joined samples' pieces are gathered into padded scratch (STAGING blob) by vd_gather_kernel and decoded by the
// kernels of mdk_decode_variants; the run columns are compacted in the SCRATCH blob.
int mdk_decode_variants_dev(int device, const uint8_t *const *seg_calls, const float *const *seg_pred_q,
                            const float *const *seg_ref_q, const int64_t *seg_rows, int64_t n_seg,
                            const int64_t *sample_seg, int64_t n_samples, int64_t max_runs, int64_t *run_sample,
                            int64_t *run_start, int64_t *run_len, float *run_pred_q, float *run_ref_q,
                            int64_t max_run_cols, uint8_t *run_pred, float *run_col_pred_q, float *run_col_ref_q,
                            float *ref_q_out, int64_t *n_runs_out, int64_t *n_run_cols_out) {
    MDK_REQUIRE(n_runs_out && n_run_cols_out, MDK_ERR_ARG, "decode_variants_dev: NULL count output");
    *n_runs_out = 0;
    *n_run_cols_out = 0;
    MDK_REQUIRE(n_seg >= 0 && n_samples >= 0 && max_runs >= 0 && max_run_cols >= 0, MDK_ERR_ARG,
                "decode_variants_dev: negative size");
    if (n_samples == 0) return MDK_OK;
    MDK_REQUIRE(seg_calls && seg_pred_q && seg_ref_q && seg_rows && sample_seg, MDK_ERR_ARG,
                "decode_variants_dev: NULL pointer");
    MDK_REQUIRE(max_runs == 0 || (run_sample && run_start && run_len && run_pred_q && run_ref_q), MDK_ERR_ARG,
                "decode_variants_dev: NULL run output");
    MDK_REQUIRE(max_run_cols == 0 || run_pred, MDK_ERR_ARG, "decode_variants_dev: NULL run column output");
    MDK_REQUIRE((run_col_pred_q == nullptr) == (run_col_ref_q == nullptr), MDK_ERR_ARG,
                "decode_variants_dev: give both run column phreds or neither");
    MDK_REQUIRE(sample_seg[0] == 0 && sample_seg[n_samples] == n_seg, MDK_ERR_ARG,
                "decode_variants_dev: sample_seg must run from 0 to n_seg");
    // padded layout: joined sample s starts at its first row + s (one padding column after each sample)
    std::vector<int64_t> pstart((size_t)n_seg), sample_pbase((size_t)n_samples + 1);
    std::vector<uint8_t> first((size_t)n_seg, 0);
    int64_t n = 0;
    for (int64_t smp = 0; smp < n_samples; ++smp) {
        MDK_REQUIRE(sample_seg[smp + 1] > sample_seg[smp], MDK_ERR_ARG, "decode_variants_dev: empty joined sample");
        sample_pbase[(size_t)smp] = n;
        first[(size_t)sample_seg[smp]] = 1;
        for (int64_t k = sample_seg[smp]; k < sample_seg[smp + 1]; ++k) {
            MDK_REQUIRE(seg_rows[k] > 0 && seg_calls[k] && seg_pred_q[k] && seg_ref_q[k], MDK_ERR_ARG,
                        "decode_variants_dev: every piece needs rows > 0 and its three pointers");
            pstart[(size_t)k] = n;
            n += seg_rows[k];
        }
        n += 1;
    }
    sample_pbase[(size_t)n_samples] = n;
    MDK_CUDA(cudaSetDevice(device));
    const int64_t n_blocks = (n + VD_THREADS - 1) / VD_THREADS;
    Staging st(Blob::STAGING, "decode_variants_dev");
    const uint8_t *const *d_calls;
    const float *const *d_spq, *const *d_srq;
    const int64_t *d_pstart, *d_rows;
    const uint8_t *d_first;
    uint8_t *d_pred, *d_mism, *d_var;
    int64_t *d_minor, *d_base, *d_rs, *d_rl, *d_tail;
    float *d_pq, *d_rq, *d_rp, *d_rr;
    st.in(&d_calls, seg_calls, n_seg);
    st.in(&d_spq, seg_pred_q, n_seg);
    st.in(&d_srq, seg_ref_q, n_seg);
    st.in(&d_pstart, pstart.data(), n_seg);
    st.in(&d_rows, seg_rows, n_seg);
    st.in(&d_first, first.data(), n_seg);
    st.take(&d_pred, n);
    st.take(&d_mism, n);
    st.take(&d_var, n);
    st.take(&d_minor, n);
    st.take(&d_pq, n);
    st.take(&d_rq, n);
    st.take(&d_base, n_blocks + 1);
    st.take(&d_tail, 2);                 // total runs (copied from d_base[n_blocks]), the bad-start flag
    st.take(&d_rs, max_runs);
    st.take(&d_rl, max_runs);
    st.take(&d_rp, max_runs);
    st.take(&d_rr, max_runs);
    if (!st.alloc()) return st.result();
    const unsigned g = (unsigned)n_blocks;
    st.check(cudaMemsetAsync(d_tail, 0, 2 * sizeof(int64_t), 0));
    vd_gather_kernel<<<g, VD_THREADS, 0, 0>>>(d_calls, d_spq, d_srq, d_pstart, d_rows, d_first, n_seg, n, d_pred,
                                              d_mism, d_minor, d_pq, d_rq, reinterpret_cast<int *>(d_tail + 1));
    vd_group_kernel<<<g, VD_THREADS, 0, 0>>>(d_minor, d_mism, n, d_var);
    vd_starts_kernel<<<g, VD_THREADS, 0, 0>>>(d_var, n, d_base);
    st.check(launch_scan_blocks(d_base, n_blocks, 0));
    vd_runs_kernel<<<g, VD_THREADS, 0, 0>>>(d_var, d_pq, d_rq, n, d_base, max_runs, d_rs, d_rl, d_rp, d_rr);
    st.check(cudaGetLastError());
    if (st.ok()) st.check(cudaMemcpyAsync(d_tail, d_base + n_blocks, sizeof(int64_t), cudaMemcpyDeviceToDevice, 0));
    int64_t tail[2] = {0, 0};
    st.out(tail, d_tail, 2);
    if (!st.ok()) return st.result();
    MDK_REQUIRE(tail[1] == 0, MDK_ERR_ARG,
                "decode_variants_dev: the first position of a sample must not be an insertion (labels.py:909-911)");
    const int64_t total = tail[0];
    *n_runs_out = total;
    if (total > max_runs) {
        set_error("decode_variants_dev: run buffers too small (see *n_runs_out)");
        return MDK_ERR_NOMEM;
    }
    st.out(run_start, d_rs, total);
    st.out(run_len, d_rl, total);
    st.out(run_pred_q, d_rp, total);
    st.out(run_ref_q, d_rr, total);
    if (!st.ok()) return st.result();
    // padded -> per-sample positions; run columns' offsets
    std::vector<int64_t> off((size_t)total + 1, 0);
    for (int64_t k = 0, smp = 0; k < total; ++k) {
        while (run_start[k] >= sample_pbase[(size_t)smp + 1]) ++smp;     // runs come in column order
        run_sample[k] = smp;
        off[(size_t)k + 1] = off[(size_t)k] + run_len[k];
    }
    const int64_t cols = off[(size_t)total];
    *n_run_cols_out = cols;
    if (cols > max_run_cols) {
        set_error("decode_variants_dev: run column buffers too small (see *n_run_cols_out)");
        return MDK_ERR_NOMEM;
    }
    if (ref_q_out)      // every real column's reference phred, padding dropped
        for (int64_t smp = 0; smp < n_samples && st.ok(); ++smp)
            st.out(ref_q_out + (sample_pbase[(size_t)smp] - smp), d_rq + sample_pbase[(size_t)smp],
                   (size_t)(sample_pbase[(size_t)smp + 1] - sample_pbase[(size_t)smp] - 1));
    if (total) {
        const bool qs = run_col_pred_q != nullptr;
        Staging sc(Blob::SCRATCH, "decode_variants_dev");
        const int64_t *d_off;
        uint8_t *d_cp;
        float *d_cpq = nullptr, *d_crq = nullptr;
        sc.in(&d_off, off.data(), total);
        sc.take(&d_cp, cols);
        if (qs) { sc.take(&d_cpq, cols); sc.take(&d_crq, cols); }
        if (!sc.alloc()) return sc.result();
        vd_run_cols_kernel<<<(unsigned)((total + VD_THREADS - 1) / VD_THREADS), VD_THREADS, 0, 0>>>(
            d_pred, d_pq, d_rq, d_rs, d_rl, d_off, total, d_cp, d_cpq, d_crq);
        sc.check(cudaGetLastError());
        sc.out(run_pred, d_cp, cols);
        if (qs) { sc.out(run_col_pred_q, d_cpq, cols); sc.out(run_col_ref_q, d_crq, cols); }
        if (!sc.ok()) return sc.result();
    }
    for (int64_t k = 0; k < total; ++k) run_start[k] -= sample_pbase[(size_t)run_sample[k]];
    return st.result();
}

}  // extern "C"
