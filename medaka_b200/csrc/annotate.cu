// Read support of variant records - `medaka tools annotate` (medaka/vcf.py:1158-1302): DP / DPS from the pileup counts at
// each variant's major column, and with spanning reads (--dpsp) DPSP, SR, AR and SC from exact affine Smith-Waterman
// scores of every spanning read against every padded haplotype of its variant.
//
// One call handles one chunk of one contig.  The records arrive in the packed form of the pileup kernels (sorted by
// position), the contig as bytes, the haplotypes as (variant geometry, allele bytes): the padded haplotypes themselves
// are never materialised, each alignment reads flank bytes and allele bytes where it needs them.
//   1. ann_trim_kernel   one warp per variant walks the CIGARs of its candidate records (those that can span the padded
//                        window, found on the host from the sorted positions) and appends the (variant, record, qstart,
//                        qend) pairs of the reads trim_read keeps (src/medaka_trimbam.c:101-246, partial = false).
//   2. ann_align_kernel  one warp per pair, persistent over the pair list: the trimmed read is striped over the lanes
//                        (one row per lane per 32-row stripe), the haplotype flows down the lanes one column per step
//                        (anti-diagonal wavefront, shuffles), the stripe's last row goes to a per-warp boundary row in
//                        global memory, 32 columns per store.  Every haplotype of the variant in turn; lane 0 adds the
//                        per-(haplotype, strand) score and best-haplotype counts with integer atomics (exact, so the sums
//                        do not depend on the order the warps finish).
//   3. ann_depth_kernel  the pileup counts of the chunk (pileup_counts_dev, the featuriser's kernels) read at each
//                        variant's major column.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace mdk {

namespace {

constexpr int ANN_NEG = -(1 << 28);       // -inf of the gap matrices (far from int32 overflow after any subtraction)
constexpr unsigned FULL = 0xffffffffu;

struct VarGeom {
    int32_t left_start, left_len;          // contig coordinate of the padded window and the length of its left flank
    int32_t right_start, right_len;        // first base after REF and the length of the right flank
    int64_t hap_lo, hap_hi;                // the variant's haplotypes (REF first) in allele_off
};

// htslib's seq_nt16 code of a sequence byte; any byte outside "=ACMGRSVTWYHKDBN" (either case) is N
__device__ __forceinline__ int nt16(uint8_t c) {
    switch (c | 0x20) {
        case 'a': return 1;
        case 'c': return 2;
        case 'm': return 3;
        case 'g': return 4;
        case 'r': return 5;
        case 's': return 6;
        case 'v': return 7;
        case 't': return 8;
        case 'w': return 9;
        case 'y': return 10;
        case 'h': return 11;
        case 'k': return 12;
        case 'd': return 13;
        case 'b': return 14;
        default: return c == '=' ? 0 : 15;
    }
}

// trim_read (src/medaka_trimbam.c:101-246) with partial = false, per operation instead of per base: the read must start
// at or before rstart and have an aligned base at or past rend; a boundary inside a deletion takes the base before;
// N or any operation outside M I D S H = X rejects the read.
__device__ bool trim_read(const uint32_t *cig, int64_t n_ops, int32_t pos, int32_t rstart, int32_t rend, int32_t *qs,
                          int32_t *qe) {
    if (pos > rstart) return false;
    bool found_s = false, found_e = false;
    int32_t qstart = -1, qend = -1, read_pos = 0, ref_pos = pos;
    for (int64_t k = 0; k < n_ops; ++k) {
        const int32_t l = (int32_t)(cig[k] >> 4);
        switch (cig[k] & 15) {
            case 0: case 7: case 8:        // M = X
                if (l > 0) {
                    if (!found_s) {
                        if (rstart >= ref_pos && rstart < ref_pos + l) { qstart = read_pos + (rstart - ref_pos); found_s = true; }
                        else if (ref_pos > rstart) { qstart = read_pos - 1; found_s = true; }
                    }
                    if (!found_e) {
                        if (rend >= ref_pos && rend < ref_pos + l) { qend = read_pos + (rend - ref_pos); found_e = true; }
                        else if (ref_pos > rend) { qend = read_pos - 1; found_e = true; }
                    }
                }
                read_pos += l;
                ref_pos += l;
                break;
            case 2: ref_pos += l; break;             // D
            case 1: case 4: read_pos += l; break;    // I S
            case 5: break;                           // H
            default: return false;                   // N (medaka_trimbam.c:183-187), P and invalid codes (:194-196)
        }
    }
    *qs = qstart;
    *qe = qend;
    return found_s && found_e && qstart >= 0 && qend >= 0;
}

__global__ void __launch_bounds__(256) ann_trim_kernel(int64_t n_var, const VarGeom *__restrict__ vg,
                                                       const int64_t *__restrict__ cand_lo,
                                                       const int64_t *__restrict__ cand_hi, Records d, int min_mapq,
                                                       int4 *__restrict__ pairs, unsigned long long *__restrict__ n_pairs) {
    const int lane = threadIdx.x & 31;
    const int64_t v = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (v >= n_var) return;
    const VarGeom g = vg[v];
    const int32_t rstart = g.left_start, rend = g.right_start + g.right_len;
    for (int64_t r0 = cand_lo[v]; r0 < cand_hi[v]; r0 += 32) {
        const int64_t r = r0 + lane;
        int32_t qs = 0, qe = 0;
        bool keep = false;
        if (r < cand_hi[v] && !(d.flag[r] & 0xF04) && (int)d.mapq[r] >= min_mapq) {   // src/medaka_bamiter.c:19-21
            const int64_t c0 = d.cigar_off[r];
            keep = trim_read(d.cigar + c0, d.cigar_off[r + 1] - c0, d.pos[r], rstart, rend, &qs, &qe) &&
                   qe - qs > 1 && (int64_t)qe <= 2 * (d.seq_off[r + 1] - d.seq_off[r]);       // medaka_trimbam.c:335
        }
        const unsigned ball = __ballot_sync(FULL, keep);
        if (!ball) continue;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(n_pairs, (unsigned long long)__popc(ball));
        base = __shfl_sync(FULL, base, 0);
        if (keep) pairs[base + __popc(ball & ((1u << lane) - 1))] = make_int4((int)v, (int)r, qs, qe);
    }
}

struct AlignArgs {
    const int4 *pairs;
    const unsigned long long *n_pairs;
    const VarGeom *vg;
    const int64_t *allele_off;
    const uint8_t *alleles;
    const uint8_t *contig;                 // bytes of [contig_start, ...)
    int32_t contig_start;
    const uint16_t *flag;
    const uint8_t *seq;
    const int64_t *seq_off;
    const int8_t *score;                   // [16][16] over nt16 codes
    int gap_open, gap_ext;
    int2 *bnd;                             // per warp: max_hap boundary cells (H, F)
    int64_t max_hap;
    unsigned long long *sr, *sc, *ar, *cells;   // sr / sc [hap][strand], ar [variant][strand]
};

struct HapView {
    const uint8_t *left, *allele, *right;
    int32_t left_len, allele_len, n;
};

__device__ __forceinline__ int hap_code(const HapView &h, int32_t k) {
    if (k < h.left_len) return nt16(h.left[k]);
    k -= h.left_len;
    if (k < h.allele_len) return nt16(h.allele[k]);
    return nt16(h.right[k - h.allele_len]);
}

// Local alignment score of the read (nt16 codes at seq nibbles qs .. qs + m) against one haplotype: Gotoh's recurrences
//   E[i][j] = max(E[i][j-1] - ext, H[i][j-1] - open),  F[i][j] = max(F[i-1][j] - ext, H[i-1][j] - open),
//   H[i][j] = max(0, H[i-1][j-1] + s(a_i, b_j), E[i][j], F[i][j]),  score = max H
// (a gap of length k costs open + (k - 1) ext, parasail's convention).  Every lane returns the warp's score.
__device__ int sw_score(const AlignArgs &a, const uint64_t *rows, const uint8_t *seq, int32_t qs, int32_t m,
                        const HapView &hap, int2 *bnd, int lane) {
    const int n = hap.n, open = a.gap_open, ext = a.gap_ext;
    const int n_stripes = (m + 31) >> 5;
    int best = 0;
    for (int s = 0; s < n_stripes; ++s) {
        const int i = (s << 5) + lane;
        const bool row_ok = i < m;
        int code = 15;
        if (row_ok) {
            const int32_t q = qs + i;
            const uint8_t byte = seq[q >> 1];
            code = (q & 1) ? (byte & 15) : (byte >> 4);
        }
        const uint64_t row = rows[code];               // 16 scores + 8, 4 bits each, indexed by the haplotype's code
        const bool first = s == 0, last = s == n_stripes - 1;
        int Hl = 0, El = ANN_NEG, Hdg = 0;             // H[i][j-1], E[i][j-1], H[i-1][j-1]
        int outH = 0, outF = ANN_NEG, outC = 15;       // this lane's last cell, read by the lane below next step
        int bH = 0, bF = ANN_NEG, bC = 15;             // lane k: boundary cell and haplotype code of column t0 + k
        int wH = 0, wF = 0;                            // lane k: last row's cell of column (j & ~31) + k, to store
        for (int t = 0; t < n + 31; ++t) {
            if ((t & 31) == 0) {
                const int k = t + lane;
                if (k < n) {
                    bC = hap_code(hap, k);
                    if (!first) { const int2 b = bnd[k]; bH = b.x; bF = b.y; }
                }
            }
            int inH = __shfl_up_sync(FULL, outH, 1);
            int inF = __shfl_up_sync(FULL, outF, 1);
            int inC = __shfl_up_sync(FULL, outC, 1);
            const int src = t & 31;
            const int c0 = __shfl_sync(FULL, bC, src);
            int h0 = 0, f0 = ANN_NEG;
            if (!first) {
                h0 = __shfl_sync(FULL, bH, src);
                f0 = __shfl_sync(FULL, bF, src);
            }
            if (lane == 0) { inH = h0; inF = f0; inC = c0; }
            const int j = t - lane;
            if (j >= 0 && j < n) {
                const int sub = (int)((row >> (4 * inC)) & 15) - 8;
                const int E = max(El - ext, Hl - open);
                const int F = max(inF - ext, inH - open);
                const int H = max(max(0, Hdg + sub), max(E, F));
                Hdg = inH;
                Hl = H;
                El = E;
                outH = H;
                outF = F;
                outC = inC;
                if (row_ok) best = max(best, H);
            }
            if (!last) {                               // lane 31's row is the next stripe's boundary
                const int jw = t - 31;
                const int h31 = __shfl_sync(FULL, outH, 31), f31 = __shfl_sync(FULL, outF, 31);
                if (jw >= 0 && (jw & 31) == lane) { wH = h31; wF = f31; }
                if (jw >= 0 && ((jw & 31) == 31 || jw == n - 1)) {
                    const int k = (jw & ~31) + lane;
                    if (k <= jw) bnd[k] = make_int2(wH, wF);
                }
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = max(best, __shfl_xor_sync(FULL, best, o));
    return best;
}

__global__ void __launch_bounds__(256) ann_align_kernel(AlignArgs a) {
    __shared__ uint64_t rows[16];
    if (threadIdx.x < 16) {
        uint64_t r = 0;
        for (int c = 0; c < 16; ++c) r |= (uint64_t)((a.score[threadIdx.x * 16 + c] + 8) & 15) << (4 * c);
        rows[threadIdx.x] = r;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    int2 *bnd = a.bnd + warp * a.max_hap;
    const int64_t n_pairs = (int64_t)*a.n_pairs;
    for (int64_t p = warp; p < n_pairs; p += n_warps) {
        const int4 pr = a.pairs[p];
        const VarGeom g = a.vg[pr.x];
        const int rev = (a.flag[pr.y] & 16) ? 1 : 0;
        const uint8_t *seq = a.seq + a.seq_off[pr.y];
        const int32_t m = pr.w - pr.z;
        HapView hv;
        hv.left = a.contig + (g.left_start - a.contig_start);
        hv.right = a.contig + (g.right_start - a.contig_start);
        hv.left_len = g.left_len;
        int first_score = 0, best_score = 0, best_h = 0;
        bool all_equal = true;
        unsigned long long cells = 0;
        for (int64_t h = g.hap_lo; h < g.hap_hi; ++h) {
            hv.allele = a.alleles + a.allele_off[h];
            hv.allele_len = (int32_t)(a.allele_off[h + 1] - a.allele_off[h]);
            hv.n = g.left_len + hv.allele_len + g.right_len;
            const int sc = sw_score(a, rows, seq, pr.z, m, hv, bnd, lane);
            cells += (unsigned long long)m * (unsigned long long)hv.n;
            if (lane == 0) atomicAdd(&a.sc[2 * h + rev], (unsigned long long)(long long)sc);
            if (h == g.hap_lo) {
                first_score = best_score = sc;
            } else {
                all_equal = all_equal && sc == first_score;
                if (sc > best_score) { best_score = sc; best_h = (int)(h - g.hap_lo); }    // first maximum wins
            }
        }
        if (lane == 0) {
            if (all_equal) atomicAdd(&a.ar[2 * (int64_t)pr.x + rev], 1ull);                // vcf.py:1376-1377
            else atomicAdd(&a.sr[2 * (g.hap_lo + best_h) + rev], 1ull);
            atomicAdd(a.cells, cells);
        }
    }
}

// DP and DPS: the counts row at the variant's major column ('acgtACGTdD': lower case and 'd' are the reverse strand)
__global__ void ann_depth_kernel(int64_t n_var, const int32_t *__restrict__ var_pos, const uint64_t *__restrict__ counts,
                                 const int64_t *__restrict__ major, const int64_t *__restrict__ minor, int64_t n_cols,
                                 int64_t *__restrict__ dp) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_var) return;
    const int64_t p = var_pos[v];
    int64_t lo = 0, hi = n_cols;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (major[mid] < p) lo = mid + 1; else hi = mid;
    }
    int64_t fwd = 0, rev = 0;
    if (lo < n_cols && major[lo] == p && minor[lo] == 0) {
        const uint64_t *c = counts + lo * 10;
        rev = (int64_t)(c[0] + c[1] + c[2] + c[3] + c[8]);
        fwd = (int64_t)(c[4] + c[5] + c[6] + c[7] + c[9]);
    }
    dp[3 * v] = fwd + rev;
    dp[3 * v + 1] = fwd;
    dp[3 * v + 2] = rev;
}

}  // namespace

}  // namespace mdk

using namespace mdk;

extern "C" int mdk_annotate(int device, int64_t n_rec, const int32_t *pos, const uint16_t *flag, const uint8_t *mapq,
                            const uint8_t *dtype, const uint32_t *cigar, const int64_t *cigar_off, const uint8_t *seq,
                            const int64_t *seq_off, const uint8_t *contig, int32_t contig_start, int32_t contig_n,
                            int32_t contig_len, int64_t n_var, const int32_t *var_pos, const int32_t *var_ref_len,
                            const int64_t *hap_off, const int64_t *allele_off, const uint8_t *alleles, int32_t pad,
                            int32_t min_mapq, int32_t dpsp, const int8_t *score, int32_t gap_open, int32_t gap_extend,
                            int64_t *dp_out, int64_t *sr_out, int64_t *ar_out, int64_t *sc_out, int64_t *stats_out,
                            float *kernel_ms) {
    MDK_REQUIRE(n_rec >= 0 && n_var >= 0 && pad >= 0 && contig_n >= 0 && contig_start >= 0, MDK_ERR_ARG,
                "annotate: bad sizes");
    MDK_REQUIRE(gap_open >= gap_extend && gap_extend >= 0, MDK_ERR_ARG, "annotate: needs gap_open >= gap_extend >= 0");
    if (kernel_ms) *kernel_ms = 0.f;
    if (stats_out) stats_out[0] = stats_out[1] = 0;
    if (n_var == 0) return MDK_OK;
    MDK_REQUIRE(var_pos && var_ref_len && hap_off && allele_off && alleles && dp_out, MDK_ERR_ARG,
                "annotate: NULL variant array");
    MDK_REQUIRE(n_rec == 0 || (pos && flag && mapq && dtype && cigar && cigar_off && seq && seq_off), MDK_ERR_ARG,
                "annotate: NULL record array");
    MDK_REQUIRE(!dpsp || (contig && score && sr_out && ar_out && sc_out), MDK_ERR_ARG, "annotate: NULL dpsp array");
    for (int64_t r = 1; r < n_rec; ++r)
        MDK_REQUIRE(pos[r] >= pos[r - 1], MDK_ERR_ARG, "annotate: records must be sorted by position");
    if (dpsp)
        for (int k = 0; k < 256; ++k)
            MDK_REQUIRE(score[k] >= -8 && score[k] <= 7, MDK_ERR_UNSUPPORTED, "annotate: scores must lie in [-8, 7]");
    const int64_t n_hap = hap_off[n_var];

    // padded windows (get_padded_haplotypes, vcf.py:1319-1326), candidate records and the pileup region
    std::vector<VarGeom> vg((size_t)n_var);
    std::vector<int64_t> cand_lo((size_t)n_var), cand_hi((size_t)n_var);
    int32_t max_span = 0;
    for (int64_t r = 0; r < n_rec; ++r) {
        int32_t span = 0;
        for (int64_t k = cigar_off[r]; k < cigar_off[r + 1]; ++k) {
            const uint32_t op = cigar[k] & 15;
            if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) span += (int32_t)(cigar[k] >> 4);
        }
        max_span = std::max(max_span, span);
    }
    int32_t pmin = INT32_MAX, pmax = 0;
    int64_t n_cand = 0, max_hap = 1;
    for (int64_t v = 0; v < n_var; ++v) {
        const int32_t p = var_pos[v], rl = var_ref_len[v];
        MDK_REQUIRE(p >= 0 && rl >= 0 && (int64_t)p + rl <= contig_len && hap_off[v + 1] > hap_off[v], MDK_ERR_ARG,
                    "annotate: variant outside its contig or without alleles");
        VarGeom &g = vg[(size_t)v];
        g.left_start = std::max(0, p - pad);
        g.left_len = p - g.left_start;
        g.right_start = p + rl;
        g.right_len = (int32_t)std::min<int64_t>((int64_t)contig_len, (int64_t)g.right_start + pad) - g.right_start;
        g.hap_lo = hap_off[v];
        g.hap_hi = hap_off[v + 1];
        pmin = std::min(pmin, p);
        pmax = std::max(pmax, p);
        if (!dpsp) continue;
        MDK_REQUIRE(g.left_start >= contig_start && g.right_start + g.right_len <= contig_start + contig_n, MDK_ERR_ARG,
                    "annotate: contig bytes do not cover a padded window");
        for (int64_t h = g.hap_lo; h < g.hap_hi; ++h)
            max_hap = std::max(max_hap, (int64_t)g.left_len + g.right_len + (allele_off[h + 1] - allele_off[h]));
        // a spanning read starts at or before the window and has an aligned base at or past its end
        const int32_t rend = g.right_start + g.right_len;
        cand_lo[(size_t)v] = std::lower_bound(pos, pos + n_rec, (int32_t)std::max<int64_t>(0, (int64_t)rend + 1 - max_span)) - pos;
        cand_hi[(size_t)v] = std::upper_bound(pos, pos + n_rec, g.left_start) - pos;
        cand_lo[(size_t)v] = std::min(cand_lo[(size_t)v], cand_hi[(size_t)v]);
        n_cand += cand_hi[(size_t)v] - cand_lo[(size_t)v];
    }

    MDK_CUDA(cudaSetDevice(device));
    int sms = 0, per_sm = 0;
    MDK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    MDK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ann_align_kernel, 256, 0));
    // persistent alignment warps: one resident wave, fewer when the boundary rows of very long haplotypes would pass
    // 256 MiB
    int64_t align_blocks = (int64_t)sms * std::max(per_sm, 1);
    align_blocks = std::max<int64_t>(1, std::min<int64_t>(align_blocks, (int64_t(1) << 28) / (8 * 8 * max_hap)));
    const int64_t n_ops = n_rec ? cigar_off[n_rec] : 0;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    if (kernel_ms) {
        MDK_CUDA(cudaEventCreate(&ev[0]));
        MDK_CUDA(cudaEventCreate(&ev[1]));
    }
    int rc = MDK_OK;
    int64_t max_cols = std::max<int64_t>(2 * ((int64_t)pmax + 1 - pmin), 16);   // medaka_counts.c:245
    for (int attempt = 0; attempt < 2; ++attempt) {
        Staging st(Blob::STAGING, "annotate");
        Records d{};
        if (n_rec) {
            st.in(&d.pos, pos, n_rec);
            st.in(&d.flag, flag, n_rec);
            st.in(&d.mapq, mapq, n_rec);
            st.in(&d.dtype, dtype, n_rec);
            st.in(&d.cigar, cigar, n_ops);
            st.in(&d.cigar_off, cigar_off, n_rec + 1);
            st.in(&d.seq, seq, seq_off[n_rec]);
            st.in(&d.seq_off, seq_off, n_rec + 1);
        }
        const int32_t *d_var_pos;
        const VarGeom *d_vg;
        const int64_t *d_lo, *d_hi, *d_aoff;
        const uint8_t *d_alleles, *d_contig;
        const int8_t *d_score;
        uint64_t *d_counts;
        int64_t *d_major, *d_minor, *d_dp;
        unsigned long long *d_red;     // sr, sc [n_hap][2], ar [n_var][2], cells, n_pairs
        st.in(&d_var_pos, var_pos, n_var);
        st.in(&d_vg, vg.data(), n_var);
        st.take(&d_counts, max_cols * 10);
        st.take(&d_major, max_cols);
        st.take(&d_minor, max_cols);
        st.take(&d_dp, 3 * n_var);
        const int64_t n_red = 4 * n_hap + 2 * n_var + 2;
        if (dpsp) {
            st.in(&d_lo, cand_lo.data(), n_var);
            st.in(&d_hi, cand_hi.data(), n_var);
            st.in(&d_aoff, allele_off, n_hap + 1);
            st.in(&d_alleles, alleles, std::max<int64_t>(allele_off[n_hap], 1));
            st.in(&d_contig, contig, std::max<int32_t>(contig_n, 1));
            st.in(&d_score, score, 256);
            st.take(&d_red, n_red);
        }
        if (!st.alloc()) { rc = st.result(); break; }
        if (kernel_ms) st.check(cudaEventRecord(ev[0], 0));
        int64_t n_cols = 0;
        rc = pileup_counts_dev(n_rec, d, n_ops, pmin, pmax + 1, 1, min_mapq, max_cols, d_counts, d_major, d_minor, &n_cols,
                               0);
        if (rc) break;
        if (n_cols > max_cols && attempt == 0) {   // a column per insertion beyond the first guess: once more, with room
            max_cols = n_cols;
            continue;
        }
        ann_depth_kernel<<<(unsigned)((n_var + 255) / 256), 256>>>(n_var, d_var_pos, d_counts, d_major, d_minor, n_cols,
                                                                    d_dp);
        st.check(cudaGetLastError());
        if (dpsp) {
            Staging sc(Blob::SCRATCH, "annotate alignments");
            int4 *d_pairs;
            int2 *d_bnd;
            sc.take(&d_pairs, std::max<int64_t>(n_cand, 1));
            sc.take(&d_bnd, align_blocks * 8 * max_hap);
            if (!sc.alloc()) { rc = sc.result(); break; }
            unsigned long long *sr = d_red, *scs = d_red + 2 * n_hap, *ar = d_red + 4 * n_hap;
            unsigned long long *cells = ar + 2 * n_var, *n_pairs = cells + 1;
            st.check(cudaMemsetAsync(d_red, 0, n_red * sizeof(unsigned long long), 0));
            if (n_cand) {
                ann_trim_kernel<<<(unsigned)((n_var * 32 + 255) / 256), 256>>>(n_var, d_vg, d_lo, d_hi, d, min_mapq,
                                                                               d_pairs, n_pairs);
                st.check(cudaGetLastError());
                AlignArgs a;
                a.pairs = d_pairs; a.n_pairs = n_pairs; a.vg = d_vg; a.allele_off = d_aoff; a.alleles = d_alleles;
                a.contig = d_contig; a.contig_start = contig_start; a.flag = d.flag; a.seq = d.seq; a.seq_off = d.seq_off;
                a.score = d_score; a.gap_open = gap_open; a.gap_ext = gap_extend; a.bnd = d_bnd; a.max_hap = max_hap;
                a.sr = sr; a.sc = scs; a.ar = ar; a.cells = cells;
                ann_align_kernel<<<(unsigned)align_blocks, 256>>>(a);
                st.check(cudaGetLastError());
            }
            if (kernel_ms) st.check(cudaEventRecord(ev[1], 0));
            st.out(sr_out, (const int64_t *)sr, 2 * n_hap);
            st.out(sc_out, (const int64_t *)scs, 2 * n_hap);
            st.out(ar_out, (const int64_t *)ar, 2 * n_var);
            if (stats_out) st.out(stats_out, (const int64_t *)cells, 2);      // cells, pairs
        } else if (kernel_ms) {
            st.check(cudaEventRecord(ev[1], 0));
        }
        st.out(dp_out, d_dp, 3 * n_var);
        if (kernel_ms && st.ok()) st.check(cudaEventElapsedTime(kernel_ms, ev[0], ev[1]));
        rc = st.result();
        break;
    }
    if (ev[0]) cudaEventDestroy(ev[0]);
    if (ev[1]) cudaEventDestroy(ev[1]);
    return rc;
}
