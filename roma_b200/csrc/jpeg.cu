// JPEG decoding on the device (roma_b200/jpeg.py), restating libjpeg-turbo's default decompression bit for bit:
//   find_end / count / chunk_scan / compact   unstuff the entropy-coded segment in parallel over bytes (FF 00 -> FF, fill FFs
//            dropped), record where every restart interval starts in the compacted stream, check RSTn runs 0..7,0.. and that
//            the first other marker is EOI;
//   sync     self-synchronising Huffman decode (after Weissenberger & Schmidt, ICPP 2018): every restart interval is cut into
//            JPG_SUBSEQ_BITS-bit subsequences, one thread each.  The decoder state at a codeword boundary is (bit offset,
//            block slot in the MCU, coefficient index k).  A pass decodes every codeword that starts in a subsequence's range
//            from the exit state its predecessor produced in the previous pass (the first subsequence of an interval starts
//            exact; in pass 0 the others guess slot 0, k 0) and records its exit state and the blocks it started.  Passes
//            repeat until no exit state changes; after p passes the first p subsequences of every interval are exact, so the
//            fixed point is the sequential decode.  One cooperative kernel runs the passes with a device-wide barrier; a
//            subsequence whose input state is the one of the previous pass keeps its exit state without decoding again, and a
//            batch that has not converged after JPG_MAX_PASSES passes is declined (ST_SYNC).
//   The IDCT declines a block outside the range where Pillow's 16-bit SIMD IDCT and the C arithmetic agree (ST_RANGE).
//   slot_scan + emit   blocks-per-subsequence scanned per interval give each subsequence its first block; a final decode
//            writes the coefficients (natural order, int16) and the raw DC differences; a decode error inside a real block,
//            bits past the interval's end or a missing block set the image's status;
//   dc       segmented scan of the DC differences per restart interval and component (exact integer work, no atomics);
//   idct     dequantise + jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, range_limit[x & RANGE_MASK]) into padded planes;
//   color    h2v1 / h2v2 fancy upsampling (replication for components <= 2 samples wide) + ycc_rgb_convert -> uint8 [H,W,C].
#include "common.cuh"
#include "tma.cuh"      // sm_count() sizes the cooperative grid

namespace rb {
namespace {

constexpr int JPG_SUBSEQ_BITS = 512;        // jpeg.py SUBSEQ_BITS
constexpr int JPG_CHUNK = 4096;             // jpeg.py CHUNK_BYTES
constexpr int JPG_THREADS = 256;            // unstuff CTAs: 16 bytes per thread
constexpr int JPG_BYTES_PER_THREAD = JPG_CHUNK / JPG_THREADS;
constexpr int SYNC_THREADS = 128;
constexpr int LUT_BITS = 9;
constexpr int TAB_INTS = (1 << LUT_BITS) + 18 + 18 + 256;
constexpr int IMG_TAB_INTS = 6 * TAB_INTS + 3 * 64;
constexpr int DESC = 64;
enum {
    D_STREAM_OFF, D_STREAM_LEN, D_COMP_OFF, D_N_INTERVALS, D_IV_OFF, D_SLOT_OFF, D_N_SLOTS, D_CHUNK_OFF, D_N_CHUNKS,
    D_BLOCK_OFF, D_N_BLOCKS, D_MCUS_PER_IV, D_BPM, D_MCUS_X, D_MCUS_Y, D_TOTAL_MCUS, D_WIDTH, D_HEIGHT, D_NCOMP,
    D_OUT_OFF, D_OUT_CH, D_SINGLE
};
constexpr int D_PLANE_OFF = 24, D_PLANE_PITCH = 28, D_HSAMP = 36, D_VSAMP = 40, D_SLOT_COMP = 44;
enum { S_END, S_STATUS, S_LEN, S_RST, S_DONE };
constexpr int ST_DATA = 1, ST_RST = 2, ST_END = 4, ST_SYNC = 8, ST_RANGE = 16, ST_SIZE = 32;
constexpr int64_t JPG_MAX_STREAM = 1LL << 29;   // bit offsets are uint32: streams up to 512 MB
constexpr int JPG_MAX_PASSES = 4096;            // sync passes before the batch is declined (ST_SYNC)
// Pillow's libjpeg-turbo runs the SIMD jpeg_idct_islow: 16-bit lanes for the dequantised coefficients, the pass-1 workspace and
// their pairwise sums, saturating packs at the end.  It equals the C arithmetic restated here while every dequantised
// coefficient and pass-1 output lies in [-IDCT_LANE, IDCT_LANE) and every pass-2 output in [-IDCT_OUT, IDCT_OUT); outside,
// the image is declined (ST_RANGE).  oracle/jpeg_decode.py states the same bound.
constexpr int64_t IDCT_LANE = 16384, IDCT_OUT = 512;
constexpr unsigned long long UNKNOWN = ~0ull;

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// byte i of an image's entropy-coded segment; outside [0, len) a value that is neither 00, FF nor a marker code
__device__ __forceinline__ int byte_at(const uint8_t* s, int64_t len, int64_t i) { return (i >= 0 && i < len) ? s[i] : 0x100; }

__device__ __forceinline__ bool is_rst(int b) { return (b & 0xF8) == 0xD0; }

// kept in the compacted stream: not a marker prefix / fill byte, not a stuffed zero or a marker code
__device__ __forceinline__ bool keep_byte(int p, int b, int nx) { return !(b == 0xFF && nx != 0) && !(p == 0xFF && b != 0xFF); }

// exclusive scan of two ints over the CTA (NT threads); totals in *tot
template <int NT>
__device__ int2 block_scan2(int2 v, int2* tot) {
    __shared__ int2 ws[NT / 32 + 1];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int2 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, inc.x, d), y = __shfl_up_sync(0xffffffffu, inc.y, d);
        if (lane >= d) inc.x += x, inc.y += y;
    }
    if (lane == 31) ws[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int2 w = lane < NT / 32 ? ws[lane] : make_int2(0, 0);
        int2 wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int x = __shfl_up_sync(0xffffffffu, wi.x, d), y = __shfl_up_sync(0xffffffffu, wi.y, d);
            if (lane >= d) wi.x += x, wi.y += y;
        }
        if (lane < NT / 32) ws[lane] = make_int2(wi.x - w.x, wi.y - w.y);
        if (lane == NT / 32 - 1) ws[NT / 32] = wi;
    }
    __syncthreads();
    const int2 base = ws[wid];
    *tot = ws[NT / 32];
    __syncthreads();
    return make_int2(base.x + inc.x - v.x, base.y + inc.y - v.y);
}

// ---- stage 1: unstuff ---------------------------------------------------------------------------------------------------
__global__ void jpg_init_kernel(rb_jpeg_args a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.batch) return;
    int32_t* st = a.state + 8 * b;
    const int64_t len = a.desc[(int64_t)b * DESC + D_STREAM_LEN];
    st[S_END] = (int32_t)len;
    st[S_STATUS] = len >= JPG_MAX_STREAM ? ST_SIZE : 0;
    st[S_LEN] = st[S_RST] = st[S_DONE] = 0;
}

__global__ void __launch_bounds__(JPG_THREADS) jpg_find_end_kernel(rb_jpeg_args a) {
    const int img = blockIdx.y;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    if (blockIdx.x >= d[D_N_CHUNKS]) return;
    const uint8_t* s = a.stream + d[D_STREAM_OFF];
    const int64_t len = d[D_STREAM_LEN];
    const int64_t i0 = (int64_t)blockIdx.x * JPG_CHUNK + threadIdx.x * JPG_BYTES_PER_THREAD;
    int64_t best = len;
    for (int t = 0; t < JPG_BYTES_PER_THREAD; ++t) {
        const int64_t i = i0 + t;
        if (i >= len) break;
        const int b = s[i];
        if (byte_at(s, len, i - 1) == 0xFF && b != 0 && b != 0xFF && !is_rst(b)) { best = i - 1; break; }
    }
    if (best < len) atomicMin(a.state + 8 * img + S_END, (int32_t)best);
}

__global__ void __launch_bounds__(JPG_THREADS) jpg_count_kernel(rb_jpeg_args a) {
    const int img = blockIdx.y;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    if (blockIdx.x >= d[D_N_CHUNKS]) return;
    const uint8_t* s = a.stream + d[D_STREAM_OFF];
    const int64_t len = d[D_STREAM_LEN], end = a.state[8 * img + S_END];
    const int64_t i0 = (int64_t)blockIdx.x * JPG_CHUNK + threadIdx.x * JPG_BYTES_PER_THREAD;
    int2 c = make_int2(0, 0);
    for (int t = 0; t < JPG_BYTES_PER_THREAD; ++t) {
        const int64_t i = i0 + t;
        if (i >= end) break;
        const int p = byte_at(s, len, i - 1), b = s[i], nx = byte_at(s, len, i + 1);
        c.x += keep_byte(p, b, nx);
        c.y += (p == 0xFF && is_rst(b));
    }
    int2 tot;
    block_scan2<JPG_THREADS>(c, &tot);
    if (threadIdx.x == 0) {
        int32_t* ch = a.chunks + 2 * (d[D_CHUNK_OFF] + blockIdx.x);
        ch[0] = tot.x;
        ch[1] = tot.y;
    }
}

// one CTA per image: exclusive scan of the chunk counts, totals, EOI / RST-count checks, interval table ends, stream padding
__global__ void __launch_bounds__(1024) jpg_chunk_scan_kernel(rb_jpeg_args a) {
    const int img = blockIdx.x;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    const int64_t nch = d[D_N_CHUNKS];
    int32_t* ch = a.chunks + 2 * d[D_CHUNK_OFF];
    int2 carry = make_int2(0, 0);
    for (int64_t k0 = 0; k0 < nch; k0 += 1024) {
        const int64_t k = k0 + threadIdx.x;
        const int2 v = k < nch ? make_int2(ch[2 * k], ch[2 * k + 1]) : make_int2(0, 0);
        int2 tot;
        const int2 ex = block_scan2<1024>(v, &tot);
        if (k < nch) ch[2 * k] = carry.x + ex.x, ch[2 * k + 1] = carry.y + ex.y;
        carry.x += tot.x;
        carry.y += tot.y;
    }
    int32_t* st = a.state + 8 * img;
    uint8_t* comp = a.comp + d[D_COMP_OFF];
    if (threadIdx.x < 16) comp[carry.x + threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        const uint8_t* s = a.stream + d[D_STREAM_OFF];
        const int64_t len = d[D_STREAM_LEN], end = st[S_END];
        const int64_t niv = d[D_N_INTERVALS];
        int status = 0;
        if (end >= len || byte_at(s, len, end + 1) != 0xD9) status |= ST_END;
        if (carry.y != niv - 1) status |= ST_RST;
        st[S_LEN] = carry.x;
        st[S_RST] = carry.y;
        if (status) atomicOr(st + S_STATUS, status);
        int32_t* iv = a.istart + d[D_IV_OFF];
        iv[0] = 0;
        iv[niv] = carry.x;
    }
}

__global__ void __launch_bounds__(JPG_THREADS) jpg_compact_kernel(rb_jpeg_args a) {
    const int img = blockIdx.y;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    if (blockIdx.x >= d[D_N_CHUNKS]) return;
    const uint8_t* s = a.stream + d[D_STREAM_OFF];
    const int64_t len = d[D_STREAM_LEN], end = a.state[8 * img + S_END], niv = d[D_N_INTERVALS];
    const int64_t i0 = (int64_t)blockIdx.x * JPG_CHUNK + threadIdx.x * JPG_BYTES_PER_THREAD;
    unsigned keep = 0, rst = 0;
    int2 c = make_int2(0, 0);
    for (int t = 0; t < JPG_BYTES_PER_THREAD; ++t) {
        const int64_t i = i0 + t;
        if (i >= end) break;
        const int p = byte_at(s, len, i - 1), b = s[i], nx = byte_at(s, len, i + 1);
        if (keep_byte(p, b, nx)) keep |= 1u << t, c.x++;
        if (p == 0xFF && is_rst(b)) rst |= 1u << t, c.y++;
    }
    int2 tot;
    const int2 ex = block_scan2<JPG_THREADS>(c, &tot);
    const int32_t* ch = a.chunks + 2 * (d[D_CHUNK_OFF] + blockIdx.x);
    int64_t pos = (int64_t)ch[0] + ex.x;
    int64_t r = (int64_t)ch[1] + ex.y;
    uint8_t* comp = a.comp + d[D_COMP_OFF];
    int32_t* iv = a.istart + d[D_IV_OFF];
    int bad = 0;
    for (int t = 0; t < JPG_BYTES_PER_THREAD; ++t) {
        if (keep >> t & 1) comp[pos++] = s[i0 + t];
        if (rst >> t & 1) {
            if (r < niv - 1) iv[r + 1] = (int32_t)pos;
            if ((s[i0 + t] & 7) != (r & 7)) bad = 1;
            ++r;
        }
    }
    if (bad) atomicOr(a.state + 8 * img + S_STATUS, ST_RST);
}

// ---- stage 2/3: Huffman decode ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t peek32(const uint8_t* p, uint32_t pos) {
    const uint8_t* q = p + (pos >> 3);
    const uint64_t w = ((uint64_t)q[0] << 32) | ((uint64_t)q[1] << 24) | ((uint64_t)q[2] << 16) | ((uint64_t)q[3] << 8) | q[4];
    return (uint32_t)(w >> (8 - (pos & 7)));
}

// symbol of the code at the top of w (len = its length), -1 for an invalid code (jpeg_huff_decode's maxcode walk)
__device__ __forceinline__ int huff_decode(const int32_t* __restrict__ t, uint32_t w, int& len) {
    const int e = t[w >> (32 - LUT_BITS)];
    if (e) {
        len = e >> 8;
        return e & 255;
    }
    const int32_t* maxcode = t + (1 << LUT_BITS);
    const int32_t* valoff = maxcode + 18;
    const int32_t* vals = valoff + 18;
    for (int l = LUT_BITS + 1; l <= 16; ++l) {
        const int code = (int)(w >> (32 - l));
        if (code <= maxcode[l]) {
            len = l;
            const int idx = code + valoff[l];
            return (idx >= 0 && idx < 256) ? vals[idx] : -1;
        }
    }
    return -1;
}

__device__ __forceinline__ int extend(uint32_t r, int s) { return r < (1u << (s - 1)) ? (int)r - (1 << s) + 1 : (int)r; }

struct Img {
    const uint8_t* bits;      // compacted stream
    const int32_t* tab;       // Huffman lookups of the image
    const int64_t* d;
    int bpm;
};

// one codeword at (pos, slot, k) -- a DC code + its extra bits, or an AC code + its extra bits -- as jdhuff.c decode_mcu does;
// false on an invalid code or a run past coefficient 63.  `ended` = the codeword finished a block.
template <bool EMIT>
__device__ __forceinline__ bool step(const Img& im, uint32_t& pos, int& slot, int& k, bool& ended, int16_t* blk) {
    const int sc = (int)(im.d[D_SLOT_COMP + slot] >> 12);
    const uint32_t w = peek32(im.bits, pos);
    int len = 0;
    ended = false;
    if (k == 0) {
        const int s = huff_decode(im.tab + (2 * sc) * TAB_INTS, w, len);
        if (s < 0) return false;
        int v = 0;
        if (s) v = extend((w << len) >> (32 - s), s);
        if (EMIT) blk[0] = (int16_t)v;
        pos += len + s;
        k = 1;
    } else {
        const int rs = huff_decode(im.tab + (2 * sc + 1) * TAB_INTS, w, len);
        if (rs < 0) return false;
        const int r = rs >> 4, s = rs & 15;
        if (s) {
            k += r;
            if (k > 63) return false;
            if (EMIT) blk[c_zigzag[k]] = (int16_t)extend((w << len) >> (32 - s), s);
            pos += len + s;
            ++k;
        } else if (r == 15) {
            k += 16;
            if (k > 64) return false;
            pos += len;
        } else {
            k = 64;                 // EOB (libjpeg ends the block on any r != 15 with s == 0)
            pos += len;
        }
    }
    if (k >= 64) {
        k = 0;
        slot = slot + 1 == im.bpm ? 0 : slot + 1;
        ended = true;
    }
    return true;
}

__device__ __forceinline__ uint64_t pack(uint32_t pos, int slot, int k) { return ((uint64_t)pos << 16) | ((uint64_t)slot << 8) | (uint64_t)k; }

// where global subsequence g lies: image, interval, bit ranges.  false for images whose stage 1 already failed.
struct Slot {
    int img;
    int64_t s, j;
    uint32_t rs, re, ivs, ive;
    bool first;
};

__device__ __forceinline__ bool locate(const rb_jpeg_args& a, int64_t g, Slot& c) {
    int lo = 0, hi = a.batch - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.desc[(int64_t)mid * DESC + D_SLOT_OFF] <= g) lo = mid; else hi = mid - 1;
    }
    const int64_t* d = a.desc + (int64_t)lo * DESC;
    c.img = lo;
    c.s = g - d[D_SLOT_OFF];
    if (c.s >= d[D_N_SLOTS] || a.state[8 * lo + S_STATUS] != 0) return false;
    const int32_t* iv = a.istart + d[D_IV_OFF];
    int64_t jl = 0, jh = d[D_N_INTERVALS] - 1;
    while (jl < jh) {
        const int64_t mid = (jl + jh + 1) >> 1;
        if (mid + (int64_t)iv[mid] * 8 / JPG_SUBSEQ_BITS <= c.s) jl = mid; else jh = mid - 1;
    }
    c.j = jl;
    c.ivs = (uint32_t)iv[jl] * 8u;
    c.ive = (uint32_t)iv[jl + 1] * 8u;
    const int64_t cell = c.s - jl;
    const int64_t lo_b = cell * JPG_SUBSEQ_BITS, hi_b = lo_b + JPG_SUBSEQ_BITS;
    c.re = (uint32_t)min((int64_t)c.ive, hi_b);
    c.rs = (uint32_t)min(max((int64_t)c.ivs, lo_b), (int64_t)c.re);
    c.first = cell == c.ivs / JPG_SUBSEQ_BITS;
    return true;
}

__device__ __forceinline__ Img image_of(const rb_jpeg_args& a, int img) {
    Img im;
    im.d = a.desc + (int64_t)img * DESC;
    im.bits = a.comp + im.d[D_COMP_OFF];
    im.tab = a.tables + (int64_t)img * IMG_TAB_INTS;
    im.bpm = (int)im.d[D_BPM];
    return im;
}

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        __threadfence();
        atomicAdd(counter, 1u);
        unsigned int seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
        __threadfence();
    }
    __syncthreads();
}

__global__ void __launch_bounds__(SYNC_THREADS, 8) jpg_sync_kernel(rb_jpeg_args a, int max_passes) {
    unsigned int target = 0;
    unsigned int* counter = (unsigned int*)(a.flags + 4);
    const int64_t stride = (int64_t)gridDim.x * SYNC_THREADS;
    int pass = 0;
    for (;; ++pass) {
        int* chg = a.flags + pass % 3;
        if (blockIdx.x == 0 && threadIdx.x == 0) a.flags[(pass + 1) % 3] = 0;
        // exit states of passes p (written), p - 1 (this pass's inputs) and p - 2 (the previous pass's inputs)
        int64_t* ex_new = a.exits + (pass % 3) * a.total_slots;
        const int64_t* ex_old = a.exits + ((pass + 2) % 3) * a.total_slots;
        const int64_t* ex_old2 = a.exits + ((pass + 1) % 3) * a.total_slots;
        bool changed = false;
        for (int64_t g = (int64_t)blockIdx.x * SYNC_THREADS + threadIdx.x; g < a.total_slots; g += stride) {
            Slot c;
            if (!locate(a, g, c)) continue;
            const Img im = image_of(a, c.img);
            const uint64_t guess = pack(c.rs, 0, 0);
            uint64_t st, prev = guess;
            if (c.first) st = prev = pack(c.ivs, 0, 0);
            else if (pass == 0) st = guess;
            else {
                st = (uint64_t)ex_old[g - 1];
                if (st == UNKNOWN) st = guess;
                if (pass >= 2) {
                    prev = (uint64_t)ex_old2[g - 1];
                    if (prev == UNKNOWN) prev = guess;
                }
            }
            if (pass > 0 && st == prev) {       // same input as the previous pass: same exit state and block count
                ex_new[g] = ex_old[g];
                continue;
            }
            uint32_t pos = (uint32_t)(st >> 16);
            int slot = (int)(st >> 8) & 255, k = (int)st & 255, cnt = 0;
            uint64_t ex;
            for (;;) {
                if (pos >= c.re) { ex = pack(pos, slot, k); break; }
                cnt += k == 0;
                bool ended;
                if (!step<false>(im, pos, slot, k, ended, nullptr) || pos > c.ive) { ex = UNKNOWN; break; }
            }
            ex_new[g] = (int64_t)ex;
            a.counts[g] = cnt;
            if (pass > 0 && (int64_t)ex != ex_old[g]) changed = true;
        }
        if (__syncthreads_or(changed) && threadIdx.x == 0) atomicOr(chg, 1);
        grid_barrier(counter, target);
        const int any = *(volatile int*)chg;
        if (pass > 0 && any == 0) break;
        if (pass + 1 >= max_passes) {
            if (blockIdx.x == 0 && threadIdx.x == 0) a.flags[5] = 1;
            break;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.flags[3] = pass + 1;
}

// first slot of interval j of an image (the slot of interval niv is the image's slot count)
__device__ __forceinline__ int64_t slot_start(const int64_t* d, const int32_t* iv, int64_t j) {
    return j >= d[D_N_INTERVALS] ? d[D_N_SLOTS] : j + (int64_t)iv[j] * 8 / JPG_SUBSEQ_BITS;
}

// one CTA per (interval, image): exclusive scan of blocks-started over the interval's subsequences
__global__ void __launch_bounds__(JPG_THREADS) jpg_slot_scan_kernel(rb_jpeg_args a) {
    const int img = blockIdx.y;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    const int64_t j = blockIdx.x;
    if (j >= d[D_N_INTERVALS] || a.state[8 * img + S_STATUS] != 0) return;
    const int32_t* iv = a.istart + d[D_IV_OFF];
    const int64_t s0 = slot_start(d, iv, j), s1 = min(slot_start(d, iv, j + 1), d[D_N_SLOTS]);
    const int32_t* cnt = a.counts + d[D_SLOT_OFF];
    int32_t* base = a.counts + a.total_slots + d[D_SLOT_OFF];
    int carry = 0;
    for (int64_t s = s0; s < s1; s += JPG_THREADS) {
        const int64_t i = s + threadIdx.x;
        const int v = i < s1 ? cnt[i] : 0;
        int2 tot;
        const int2 ex = block_scan2<JPG_THREADS>(make_int2(v, 0), &tot);
        if (i < s1) base[i] = carry + ex.x;
        carry += tot.x;
    }
}

__global__ void __launch_bounds__(SYNC_THREADS) jpg_emit_kernel(rb_jpeg_args a) {
    const int64_t g = (int64_t)blockIdx.x * SYNC_THREADS + threadIdx.x;
    if (g >= a.total_slots) return;
    Slot c;
    if (!locate(a, g, c)) return;
    const Img im = image_of(a, c.img);
    const int64_t* d = im.d;
    const int64_t* exits = a.exits + ((a.flags[3] - 1) % 3) * a.total_slots;
    const int64_t base = a.counts[a.total_slots + g];
    const int64_t R = d[D_MCUS_PER_IV];
    const int64_t nblk = min(R, d[D_TOTAL_MCUS] - c.j * R) * im.bpm;       // blocks of this interval
    int16_t* coef = a.coef + (d[D_BLOCK_OFF] + c.j * R * im.bpm) * 64;
    uint64_t st = c.first ? pack(c.ivs, 0, 0) : (uint64_t)exits[g - 1];
    int err = 0, done = 0;
    if (st == UNKNOWN) {
        err = base < nblk && c.rs < c.re;
    } else {
        uint32_t pos = (uint32_t)(st >> 16);
        int slot = (int)(st >> 8) & 255, k = (int)st & 255;
        int64_t blk = k ? base - 1 : base;
        if (blk < 0) err = 1;
        while (!err && pos < c.re && blk < nblk) {
            bool ended;
            if (!step<true>(im, pos, slot, k, ended, coef + blk * 64) || pos > c.ive) { err = 1; break; }
            if (ended) ++done, ++blk;
        }
    }
    if (err) atomicOr(a.state + 8 * c.img + S_STATUS, ST_DATA);
    if (done) atomicAdd(a.state + 8 * c.img + S_DONE, done);
}

// one CTA per (interval * 3 + scan component, image): DC[t] = sum of the differences up to block t of that component in the interval
__global__ void __launch_bounds__(JPG_THREADS) jpg_dc_kernel(rb_jpeg_args a) {
    const int img = blockIdx.y;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    int32_t* st = a.state + 8 * img;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        int bad = 0;
        if (st[S_STATUS] == 0 && st[S_DONE] != d[D_N_BLOCKS]) bad |= ST_DATA;
        if (a.flags[5]) bad |= ST_SYNC;
        if (bad) atomicOr(st + S_STATUS, bad);
    }
    const int64_t j = blockIdx.x / 3;
    const int sc = blockIdx.x % 3;
    if (j >= d[D_N_INTERVALS] || sc >= d[D_NCOMP]) return;
    const int bpm = (int)d[D_BPM];
    int off = -1, nb = 0;
    for (int s = 0; s < bpm; ++s)
        if ((int)(d[D_SLOT_COMP + s] >> 12) == sc) {
            if (off < 0) off = s;
            ++nb;
        }
    if (off < 0) return;
    const int64_t R = d[D_MCUS_PER_IV];
    const int64_t nmcu = min(R, d[D_TOTAL_MCUS] - j * R);
    int16_t* coef = a.coef + (d[D_BLOCK_OFF] + j * R * bpm) * 64;
    unsigned carry = 0;
    const int64_t n = nmcu * nb;
    for (int64_t t0 = 0; t0 < n; t0 += JPG_THREADS) {
        const int64_t t = t0 + threadIdx.x;
        int16_t* p = t < n ? coef + ((t / nb) * bpm + off + t % nb) * 64 : nullptr;
        const int v = p ? *p : 0;
        int2 tot;
        const int2 ex = block_scan2<JPG_THREADS>(make_int2(v, 0), &tot);
        if (p) *p = (int16_t)(carry + (unsigned)ex.x + (unsigned)v);
        carry += (unsigned)tot.x;
    }
}

// ---- stage 4: dequantise + ISLOW IDCT -----------------------------------------------------------------------------------
// jidctint.c with CONST_BITS 13, PASS1_BITS 2; JLONG arithmetic in 64 bits
__device__ __forceinline__ void idct8(const int64_t* x, int64_t* o) {
    int64_t z1 = (x[2] + x[6]) * 4433;
    int64_t tmp2 = z1 + x[6] * -15137, tmp3 = z1 + x[2] * 6270;
    int64_t tmp0 = (x[0] + x[4]) * 8192, tmp1 = (x[0] - x[4]) * 8192;
    const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    tmp0 = x[7]; tmp1 = x[5]; tmp2 = x[3]; tmp3 = x[1];
    z1 = tmp0 + tmp3;
    int64_t z2 = tmp1 + tmp2, z3 = tmp0 + tmp2, z4 = tmp1 + tmp3;
    const int64_t z5 = (z3 + z4) * 9633;
    tmp0 *= 2446; tmp1 *= 16819; tmp2 *= 25172; tmp3 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    o[0] = t10 + tmp3; o[7] = t10 - tmp3; o[1] = t11 + tmp2; o[6] = t11 - tmp2;
    o[2] = t12 + tmp1; o[5] = t12 - tmp1; o[3] = t13 + tmp0; o[4] = t13 - tmp0;
}

__device__ __forceinline__ int64_t descale(int64_t x, int n) { return (x + ((int64_t)1 << (n - 1))) >> n; }

// range_limit[x & RANGE_MASK] of the post-IDCT table: the 10-bit wrap, then the clamp of the centred sample
__device__ __forceinline__ uint8_t range_limit(int64_t v) {
    const int x = (int)(v & 1023);
    const int s = x < 512 ? x : x - 1024;
    return (uint8_t)min(max(s + 128, 0), 255);
}

__device__ __forceinline__ bool outside(int64_t v, int64_t lim) { return v < -lim || v >= lim; }

__device__ __forceinline__ int find_image(const int64_t* desc, int batch, int field, int64_t g) {
    int lo = 0, hi = batch - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (desc[(int64_t)mid * DESC + field] <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// 8 threads per block: column pass into shared memory, then row pass into the plane
__global__ void __launch_bounds__(256) jpg_idct_kernel(rb_jpeg_args a) {
    __shared__ int32_t ws[32][64];
    const int64_t gt = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t gb = gt >> 3;
    const int lane = threadIdx.x & 7, lb = threadIdx.x >> 3;
    const bool live = gb < a.total_blocks;
    int img = 0;
    bool ok = false;
    if (live) {
        img = find_image(a.desc, a.batch, D_BLOCK_OFF, gb);
        ok = a.state[8 * img + S_STATUS] == 0;
    }
    const int64_t* d = a.desc + (int64_t)img * DESC;
    const int64_t local = gb - d[D_BLOCK_OFF];
    int ci = 0;
    int64_t by = 0, bx = 0;
    bool bad = false;
    if (ok) {
        const int64_t mx = d[D_MCUS_X];
        if (d[D_SINGLE]) {
            ci = (int)(d[D_SLOT_COMP] & 15);
            by = local / mx;
            bx = local % mx;
        } else {
            const int bpm = (int)d[D_BPM];
            const int64_t mcu = local / bpm;
            const int sc = (int)d[D_SLOT_COMP + local % bpm];
            ci = sc & 15;
            by = (mcu / mx) * d[D_VSAMP + ci] + ((sc >> 4) & 15);
            bx = (mcu % mx) * d[D_HSAMP + ci] + ((sc >> 8) & 15);
        }
        const int16_t* cf = a.coef + gb * 64;
        const int32_t* q = a.tables + (int64_t)img * IMG_TAB_INTS + 6 * TAB_INTS + ci * 64;
        int64_t x[8], o[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            x[r] = (int64_t)((int)cf[r * 8 + lane] * (int)(int16_t)q[r * 8 + lane]);
            bad |= outside(x[r], IDCT_LANE);
        }
        idct8(x, o);
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int64_t w = descale(o[r], 13 - 2);
            bad |= outside(w, IDCT_LANE);
            ws[lb][r * 8 + lane] = (int32_t)w;
        }
    }
    __syncwarp();
    if (ok) {
        int64_t x[8], o[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) x[c] = ws[lb][lane * 8 + c];
        idct8(x, o);
        uint8_t* row = a.planes + d[D_PLANE_OFF + ci] + (by * 8 + lane) * d[D_PLANE_PITCH + ci] + bx * 8;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int64_t v = descale(o[c], 13 + 2 + 3);
            bad |= outside(v, IDCT_OUT);
            row[c] = range_limit(v);
        }
        if (bad) atomicOr(a.state + 8 * img + S_STATUS, ST_RANGE);
    }
}

// ---- stage 5: upsample + colour convert ---------------------------------------------------------------------------------
// chroma sample at output (y, x) for luma sampling (h, v) (jdsample.c h2v1 / h2v2 fancy, or replication when dw <= 2)
__device__ __forceinline__ int chroma(const uint8_t* p, int64_t pitch, int h, int v, int64_t dw, int64_t dh, int64_t y, int64_t x) {
    if (h == 1) return p[y * pitch + x];
    const int64_t j = x >> 1;
    const bool odd = x & 1;
    if (dw <= 2) return p[(v == 2 ? y >> 1 : y) * pitch + j];
    if (v == 1) {
        const uint8_t* r = p + y * pitch;
        const int c = r[j];
        if (!odd) return j == 0 ? c : (3 * c + r[j - 1] + 1) >> 2;
        return j == dw - 1 ? c : (3 * c + r[j + 1] + 2) >> 2;
    }
    const int64_t i = y >> 1;
    const int64_t i1 = min(max((y & 1) ? i + 1 : i - 1, (int64_t)0), dh - 1);
    const uint8_t* r0 = p + i * pitch;
    const uint8_t* r1 = p + i1 * pitch;
    const int c = 3 * r0[j] + r1[j];
    if (!odd) return j == 0 ? (4 * c + 8) >> 4 : (3 * c + 3 * r0[j - 1] + r1[j - 1] + 8) >> 4;
    return j == dw - 1 ? (4 * c + 7) >> 4 : (3 * c + 3 * r0[j + 1] + r1[j + 1] + 7) >> 4;
}

__global__ void __launch_bounds__(256) jpg_color_kernel(rb_jpeg_args a) {
    const int img = blockIdx.y;
    const int64_t* d = a.desc + (int64_t)img * DESC;
    const int64_t W = d[D_WIDTH], H = d[D_HEIGHT];
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= W * H || a.state[8 * img + S_STATUS] != 0) return;
    const int64_t y = i / W, x = i % W;
    const int C = (int)d[D_OUT_CH];
    uint8_t* o = a.out + d[D_OUT_OFF] + i * C;
    const int ysamp = a.planes[d[D_PLANE_OFF] + y * d[D_PLANE_PITCH] + x];
    if (d[D_NCOMP] == 1) {
        for (int c = 0; c < C; ++c) o[c] = (uint8_t)ysamp;
        return;
    }
    const int h = (int)d[D_HSAMP], v = (int)d[D_VSAMP];
    const int64_t dw = (W + h - 1) / h, dh = (H + v - 1) / v;
    const int cb = chroma(a.planes + d[D_PLANE_OFF + 1], d[D_PLANE_PITCH + 1], h, v, dw, dh, y, x);
    const int cr = chroma(a.planes + d[D_PLANE_OFF + 2], d[D_PLANE_PITCH + 2], h, v, dw, dh, y, x);
    const int xb = cb - 128, xr = cr - 128;
    const int r = ysamp + ((91881 * xr + 32768) >> 16);
    const int g = ysamp + ((-22554 * xb + 32768 - 46802 * xr) >> 16);
    const int b = ysamp + ((116130 * xb + 32768) >> 16);
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[1] = (uint8_t)min(max(g, 0), 255);
    o[2] = (uint8_t)min(max(b, 0), 255);
}

int jpg_check(const rb_jpeg_args* a, const char* what) {
    RB_REQUIRE(a && a->batch > 0 && a->stream && a->desc && a->tables && a->comp && a->chunks && a->istart && a->exits && a->counts &&
               a->coef && a->state && a->flags, "%s: null argument", what);
    RB_REQUIRE(a->total_slots > 0 && a->total_slots < (1LL << 31) && a->max_chunks > 0 && a->max_intervals > 0, "%s: bad sizes", what);
    return 0;
}

}  // namespace
}  // namespace rb

using namespace rb;

extern "C" int romab200_jpeg_entropy(const rb_jpeg_args* a, void* stream) {
    if (jpg_check(a, "jpeg_entropy")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 chunks(a->max_chunks, a->batch);
    jpg_init_kernel<<<(a->batch + 127) / 128, 128, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(init)")) return 1;
    jpg_find_end_kernel<<<chunks, JPG_THREADS, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(find end)")) return 1;
    jpg_count_kernel<<<chunks, JPG_THREADS, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(count)")) return 1;
    jpg_chunk_scan_kernel<<<a->batch, 1024, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(chunk scan)")) return 1;
    jpg_compact_kernel<<<chunks, JPG_THREADS, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(compact)")) return 1;
    // sync passes: one cooperative kernel, every CTA resident
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jpg_sync_kernel, SYNC_THREADS, 0);
    RB_REQUIRE(per_sm > 0, "jpeg_entropy: cannot size the cooperative grid");
    const int64_t want = (a->total_slots + SYNC_THREADS - 1) / SYNC_THREADS;
    const int grid = (int)std::min<int64_t>(want, (int64_t)per_sm * sm_count());
    rb_jpeg_args args = *a;
    int max_passes = (int)std::min<int64_t>(a->total_slots + 2, JPG_MAX_PASSES);
    void* kargs[] = {(void*)&args, (void*)&max_passes};
    cudaError_t err = cudaLaunchCooperativeKernel((void*)jpg_sync_kernel, dim3(grid), dim3(SYNC_THREADS), kargs, 0, st);
    RB_REQUIRE(err == cudaSuccess, "jpeg_entropy: cooperative launch failed: %s", cudaGetErrorString(err));
    if (check_launch("jpeg_entropy(sync)")) return 1;
    jpg_slot_scan_kernel<<<dim3(a->max_intervals, a->batch), JPG_THREADS, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(slot scan)")) return 1;
    jpg_emit_kernel<<<(unsigned)want, SYNC_THREADS, 0, st>>>(*a);
    if (check_launch("jpeg_entropy(emit)")) return 1;
    jpg_dc_kernel<<<dim3(a->max_intervals * 3, a->batch), JPG_THREADS, 0, st>>>(*a);
    return check_launch("jpeg_entropy(dc)");
}

extern "C" int romab200_jpeg_pixels(const rb_jpeg_args* a, void* stream) {
    if (jpg_check(a, "jpeg_pixels")) return 1;
    RB_REQUIRE(a->planes && a->out && a->max_pixels > 0 && a->total_blocks > 0, "jpeg_pixels: null output or empty batch");
    cudaStream_t st = (cudaStream_t)stream;
    jpg_idct_kernel<<<(unsigned)((a->total_blocks * 8 + 255) / 256), 256, 0, st>>>(*a);
    if (check_launch("jpeg_pixels(idct)")) return 1;
    jpg_color_kernel<<<dim3((unsigned)((a->max_pixels + 255) / 256), a->batch), 256, 0, st>>>(*a);
    return check_launch("jpeg_pixels(color)");
}
