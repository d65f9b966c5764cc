// Device-resident data-shard iterator kernels (SURVEY §8f-1).
//
// Reference: util/data.py:11-30 shard_indices (`indices[rank::world]` after the optional MT19937 shuffle and tail drop)
// and examples/mnist.py:16-21 (torchvision ToTensor + Normalize((0.1307,), (0.3081,)) + DataLoader batching, on the host).
// Here the whole uint8 dataset stays in HBM (MNIST: 47 MB of 180 GB); the epoch permutation is uploaded once per epoch
// (bit-exact host computation — the same numpy MT19937 stream the reference uses) and each step is one gather kernel:
//   out[i, :] = (float(images[idx[i], :]) / 255 - mean) / std                      784 B read, 3136 (fp32) B written / sample
// HBM-bound byte work: 16 pixels (one 128-bit load) per thread, 4x 128-bit stores, rows found through idx[] (L2-resident).
#include <cmath>

#include "dmlb_common.cuh"

namespace dmlb {

__device__ __forceinline__ float norm_px(uint32_t byte, float mean, float std) {
    // exactly torchvision's arithmetic order: ToTensor -> x/255 ; Normalize -> (x - mean) / std   (IEEE fp32 div/sub/div)
    return ((float)byte / 255.0f - mean) / std;
}

template <bool kBf16>
__global__ void __launch_bounds__(256)
shard_gather_u8_kernel(const uint8_t *__restrict__ images, const long long *__restrict__ idx, long long batch,
                       long long row_elems, long long vec_per_row, float mean, float std, void *out) {
    const long long total = batch * vec_per_row;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long i = t / vec_per_row, v = t - i * vec_per_row;
        const long long row = idx[i];
        const uint4 px = ld_stream_u4(reinterpret_cast<const uint4 *>(images + row * row_elems) + v);
        const uint32_t w[4] = {px.x, px.y, px.z, px.w};
        float f[16];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            f[4 * k + 0] = norm_px(w[k] & 0xff, mean, std);
            f[4 * k + 1] = norm_px((w[k] >> 8) & 0xff, mean, std);
            f[4 * k + 2] = norm_px((w[k] >> 16) & 0xff, mean, std);
            f[4 * k + 3] = norm_px(w[k] >> 24, mean, std);
        }
        if (kBf16) {
            uint4 *o = reinterpret_cast<uint4 *>(reinterpret_cast<uint16_t *>(out) + i * row_elems) + 2 * v;
            o[0] = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
            o[1] = make_uint4(pack_bf16x2(f[8], f[9]), pack_bf16x2(f[10], f[11]), pack_bf16x2(f[12], f[13]),
                              pack_bf16x2(f[14], f[15]));
        } else {
            float4 *o = reinterpret_cast<float4 *>(reinterpret_cast<float *>(out) + i * row_elems) + 4 * v;
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = make_float4(f[4 * k], f[4 * k + 1], f[4 * k + 2], f[4 * k + 3]);
        }
    }
}

template <bool kBf16>
__global__ void __launch_bounds__(256)
shard_gather_u8_scalar_kernel(const uint8_t *__restrict__ images, const long long *__restrict__ idx, long long batch,
                              long long row_elems, float mean, float std, void *out) {
    const long long total = batch * row_elems;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long i = t / row_elems, e = t - i * row_elems;
        float f = norm_px(images[idx[i] * row_elems + e], mean, std);
        if (kBf16)
            reinterpret_cast<uint16_t *>(out)[t] = f32_to_bf16(f);
        else
            reinterpret_cast<float *>(out)[t] = f;
    }
}

__global__ void shard_gather_i64_kernel(const long long *__restrict__ labels, const long long *__restrict__ idx,
                                        long long batch, long long *out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < batch; i += (long long)gridDim.x * blockDim.x)
        out[i] = labels[idx[i]];
}

__global__ void shard_slice_kernel(const long long *__restrict__ perm, long long first, long long count, long long rank,
                                   long long world, long long *out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
        out[i] = perm[(first + i) * world + rank];
}

static inline int grid_for(long long work, int threads) {
    long long g = (work + threads - 1) / threads;
    long long cap = (long long)sm_count() * 8;
    if (g < 1) g = 1;
    return (int)(g < cap ? g : cap);
}

// ---- colour images: gather + pad + crop + flip + per-channel normalise (dmlb_image_batch_u8) ------------------------
// One CTA job = one band of up to `rows` output rows of one sample.  The band's window rows are staged into shared memory
// as the 16-byte aligned chunks of the source rows that cover them (so the loads are 128-bit whatever the crop offset),
// then written out in the output's contiguous order, 16-byte stores for the body of every contiguous run.  Normalised
// values come from a per-launch [C][256] table in shared memory built with norm_px, so every element is two shared
// loads and no division.  HBM traffic is the window bytes (plus < 32 B of chunk rounding per row) and the output.

constexpr uint64_t kImageGamma = 0x9e3779b97f4a7c15ull;
constexpr int kImageThreads = 256;
constexpr int kImageBandBytes = 24576;  // staged window bytes per CTA (+ the 4 KB table)
constexpr int kImageCtasPerSm = 6;      // grid cap: what fits one SM at <= 40 registers per thread (ptxas -v)
constexpr int kImageMaxRowBytes = 49152;

__host__ __device__ __forceinline__ uint64_t splitmix64_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

struct ImageArgs {
    const uint8_t *images;
    const long long *idx;
    void *out;
    int *params;
    long long batch, sample_bytes;
    unsigned long long seed;
    long long epoch;
    int H, W, C, oh, ow, pad, random_crop, hflip;
    int rows, bands, rowcap;  // band height, bands per sample, staged bytes per window row
    float mean[4], std[4];
};

// The window of one sample, in padded coordinates (include/dmlb.h states the rule).
__device__ __forceinline__ void image_window(const ImageArgs &a, long long row, int &top, int &left, int &flip) {
    const int dy = a.H + 2 * a.pad - a.oh, dx = a.W + 2 * a.pad - a.ow;
    uint64_t h = splitmix64_mix(a.seed + kImageGamma);
    h = splitmix64_mix(h ^ ((uint64_t)a.epoch + kImageGamma));
    h = splitmix64_mix(h ^ ((uint64_t)row + kImageGamma));
    if (a.random_crop) {
        top = (int)(((uint64_t)(uint32_t)h * (uint64_t)(dy + 1)) >> 32);
        left = (int)(((uint64_t)(uint32_t)(h >> 32) * (uint64_t)(dx + 1)) >> 32);
    } else {  // Python round(d / 2): halves go to the even neighbour
        top = (dy >> 1) + ((dy & 1) & ((dy >> 1) & 1));
        left = (dx >> 1) + ((dx & 1) & ((dx >> 1) & 1));
    }
    flip = a.hflip ? (int)(splitmix64_mix(h + kImageGamma) >> 63) : 0;
}

// One band of one sample, staged in shared memory: window row r holds source bytes from an address whose low 4 bits are
// `head(r)` (0 on the byte-load path), columns [u_lo, u_hi) of the window are inside the image, the rest is padding.
template <bool kVecLoad>
struct ImageBand {
    const uint8_t *sm;
    const uint32_t *lut;
    uint32_t img_mod;  // low bits of the address of window column u_lo in source row 0
    int sy0, H, WC, C, ow, u_lo, u_hi, rowcap, flip;

    __device__ __forceinline__ uint32_t value(int r, int x, int c) const {
        const int u = flip ? ow - 1 - x : x;
        const int sy = sy0 + r;
        uint32_t byte = 0;
        if ((unsigned)sy < (unsigned)H && u >= u_lo && u < u_hi) {
            const uint32_t head = kVecLoad ? ((img_mod + (uint32_t)sy * (uint32_t)WC) & 15u) : 0u;
            byte = sm[r * rowcap + head + (u - u_lo) * C + c];
        }
        return lut[c * 256 + byte];
    }
};

// Walks a contiguous run of output elements in memory order: NCHW runs stay in one channel plane, NHWC runs step c fastest.
// Band: any band type with members C, ow and value(r, x, c) (ImageBand, ResampleBand).
template <class Band, bool kNHWC>
struct ImageCursor {
    const Band &b;
    int r, x, c;
    __device__ __forceinline__ uint32_t next() {
        const uint32_t v = b.value(r, x, c);
        if (kNHWC && ++c < b.C) return v;
        if (kNHWC) c = 0;
        if (++x == b.ow) x = 0, ++r;
        return v;
    }
};

// Elements [0, n) of a contiguous output run starting at element `first` of `out`; element k is produced by a cursor
// from at(k).  Scalar stores up to the first 16-byte boundary and after the last, 16-byte stores in between.
template <bool kBf16, class At>
__device__ __forceinline__ void image_store_run(void *out, long long first, int n, const At &at) {
    constexpr int E = kBf16 ? 2 : 4, V = 16 / E;
    const uintptr_t base = (uintptr_t)out + (uintptr_t)first * E;
    int head = (int)(((16u - (uint32_t)(base & 15)) & 15u) / E);
    if (head > n) head = n;
    const int nvec = (n - head) / V, tail0 = head + nvec * V, nscalar = head + (n - tail0);
    for (int t = threadIdx.x; t < nvec; t += blockDim.x) {
        auto cur = at(head + t * V);
        uint32_t w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (kBf16) {
                const uint32_t lo = cur.next();
                w[j] = lo | (cur.next() << 16);
            } else {
                w[j] = cur.next();
            }
        }
        *reinterpret_cast<uint4 *>(base + (uintptr_t)(head + t * V) * E) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    for (int t = threadIdx.x; t < nscalar; t += blockDim.x) {
        const int k = t < head ? t : tail0 + (t - head);
        const uint32_t v = at(k).next();
        if (kBf16)
            reinterpret_cast<uint16_t *>(base)[k] = (uint16_t)v;
        else
            reinterpret_cast<uint32_t *>(base)[k] = v;
    }
}

template <bool kBf16, bool kNHWC, bool kVecLoad>
__global__ void __launch_bounds__(kImageThreads) image_batch_u8_kernel(const ImageArgs a) {
    extern __shared__ uint4 s_band[];
    __shared__ uint32_t s_lut[4 * 256];
    uint8_t *sm = reinterpret_cast<uint8_t *>(s_band);
    for (int e = threadIdx.x; e < a.C * 256; e += blockDim.x) {
        const float f = norm_px(e & 255, a.mean[e >> 8], a.std[e >> 8]);
        s_lut[e] = kBf16 ? (uint32_t)f32_to_bf16(f) : __float_as_uint(f);
    }
    const long long jobs = a.batch * a.bands;
    const int WC = a.W * a.C, plane = a.oh * a.ow;
    for (long long job = blockIdx.x; job < jobs; job += gridDim.x) {
        const long long i = job / a.bands;
        const int y0 = (int)(job - i * a.bands) * a.rows;
        const int nr = min(a.rows, a.oh - y0);
        const long long row = a.idx[i];
        int top, left, flip;
        image_window(a, row, top, left, flip);
        if (a.params && y0 == 0 && threadIdx.x == 0) {
            a.params[3 * i] = top;
            a.params[3 * i + 1] = left;
            a.params[3 * i + 2] = flip;
        }
        const uint8_t *img = a.images + row * a.sample_bytes;
        const int sx0 = left - a.pad, sy0 = top - a.pad + y0;
        const int u_lo = max(0, -sx0), u_hi = min(a.ow, a.W - sx0);
        const int nbytes = (u_hi - u_lo) * a.C;
        const uint8_t *col0 = img + (long long)(sx0 + u_lo) * a.C;  // window column u_lo of source row 0
        __syncthreads();  // the previous job's readers are done with the band (and the table is complete)
        if (kVecLoad) {
            const uint8_t *img_end = img + a.sample_bytes;
            const int cpr = a.rowcap >> 4;
            for (int t = threadIdx.x; t < nr * cpr; t += blockDim.x) {
                const int r = t / cpr, j = t - r * cpr, sy = sy0 + r;
                if ((unsigned)sy >= (unsigned)a.H || nbytes <= 0) continue;
                const uint8_t *s = col0 + (long long)sy * WC;
                const uint8_t *lo = reinterpret_cast<const uint8_t *>((uintptr_t)s & ~(uintptr_t)15);
                if (j * 16 >= (int)(s - lo) + nbytes) continue;
                const uint8_t *chunk = lo + 16 * j;
                uint4 v;
                if (chunk + 16 <= img_end) {
                    v = ld_stream_u4(reinterpret_cast<const uint4 *>(chunk));
                } else {  // the sample's last chunk: never read past the tensor
                    uint8_t tmp[16];
#pragma unroll
                    for (int k = 0; k < 16; ++k) tmp[k] = chunk + k < img_end ? chunk[k] : 0;
                    v = *reinterpret_cast<uint4 *>(tmp);
                }
                reinterpret_cast<uint4 *>(sm + r * a.rowcap)[j] = v;
            }
        } else {
            for (int t = threadIdx.x; t < nr * a.rowcap; t += blockDim.x) {
                const int r = t / a.rowcap, k = t - r * a.rowcap, sy = sy0 + r;
                if ((unsigned)sy < (unsigned)a.H && k < nbytes) sm[t] = col0[(long long)sy * WC + k];
            }
        }
        __syncthreads();
        const ImageBand<kVecLoad> band{sm, s_lut, (uint32_t)(uintptr_t)col0, sy0, a.H, WC, a.C, a.ow, u_lo, u_hi,
                                       a.rowcap, flip};
        if (kNHWC) {
            const int C = a.C, ow = a.ow;
            image_store_run<kBf16>(a.out, i * plane * C + (long long)y0 * ow * C, nr * ow * C, [&](int k) {
                const int p = k / C;
                return ImageCursor<ImageBand<kVecLoad>, true>{band, p / ow, p - (p / ow) * ow, k - p * C};
            });
        } else {
            for (int c = 0; c < a.C; ++c) {
                const int ow = a.ow;
                image_store_run<kBf16>(a.out, (i * a.C + c) * plane + (long long)y0 * ow, nr * ow, [&](int k) {
                    return ImageCursor<ImageBand<kVecLoad>, false>{band, k / ow, k - (k / ow) * ow, c};
                });
            }
        }
    }
}

template <bool kBf16, bool kNHWC>
static void launch_image(bool vec_load, int grid, size_t smem, cudaStream_t st, const ImageArgs &a) {
    if (vec_load)
        image_batch_u8_kernel<kBf16, kNHWC, true><<<grid, kImageThreads, smem, st>>>(a);
    else
        image_batch_u8_kernel<kBf16, kNHWC, false><<<grid, kImageThreads, smem, st>>>(a);
}


// ---- resampled colour images: box -> antialiased bilinear resize -> window -> flip -> normalise ---------------------
// (dmlb_image_resample_u8; include/dmlb.h states the rule.)  One CTA job = one band of up to `rows` output rows of one
// sample.  The CTA builds the sample's column taps (xmin, xsize, weights) for the window's columns and the row taps of
// the band, runs the horizontal pass over the band's source rows into an fp32 [srows][out_w * C] tile in shared memory,
// then the vertical pass, written in the output's contiguous order by image_store_run.  Source bytes are read through
// L1 (a box row's bytes are read by neighbouring columns' taps) and mapped through a 256-entry fl32(byte) / 255 table.
// Every operation of the tap and pixel arithmetic is rounded once, as written (no FMA contraction).

constexpr int kResampleThreads = 256;
constexpr int kResampleMaxScale = 8;          // H <= 8 resize_h, W <= 8 resize_w: at most 2 * 8 + 1 taps per output
constexpr int kResampleMaxRowElems = 1024;    // out_w * C
constexpr int kResampleMaxSide = 32768;       // H, W, resize_h, resize_w: tap positions stay exact in fp32
constexpr int kResampleBandBytes = 32768;     // target size of a band's tile + row taps (one row may need up to 76 KB)
constexpr int kResampleCtasPerSm = 4;

struct ResampleArgs {
    const uint8_t *images;
    const long long *idx;
    const int *boxes;
    void *out;
    long long batch, sample_bytes;
    int H, W, C, rh, rw, win_top, win_left, oh, ow;
    int rows, bands, srows, kx, ky;  // band height, bands per sample, tile rows, column / row tap stride
    float mean[4], std[4];
};

// One axis of one sample: ATen's antialiased bilinear filter (aten/src/ATen/native/cpu/UpSampleKernel.cpp,
// _compute_indices_min_size_weights_aa with align_corners = false), with its C++ types: scale, support, center and the
// weights are fp32; center, the bounds and the filter argument are formed in fp64 where C++ promotes, then rounded.
struct ResampleAxis {
    float scale, support, invscale;
    int K, n_in;

    __device__ __forceinline__ ResampleAxis(int in, int out) : n_in(in) {
        scale = __fdiv_rn((float)in, (float)out);
        support = scale >= 1.0f ? scale : 1.0f;
        invscale = scale >= 1.0f ? (float)(1.0 / (double)scale) : 1.0f;
        K = (int)ceilf(support) * 2 + 1;
    }
    __device__ __forceinline__ float center(int i) const { return (float)((double)scale * ((double)i + 0.5)); }
    __device__ __forceinline__ int xmin(int i) const {
        return max((int)((double)__fsub_rn(center(i), support) + 0.5), 0);
    }
    __device__ __forceinline__ int xend(int i) const {  // one past the last tap before the clamp to K
        return min((int)((double)__fadd_rn(center(i), support) + 0.5), n_in);
    }
    // xmin and xsize of output index i; weights w[0, xsize), normalised by their fp32 sum taken in increasing j.
    __device__ __forceinline__ void taps(int i, int &x0, int &n, float *w) const {
        const float c = center(i);
        x0 = xmin(i);
        n = min(max(xend(i) - x0, 0), K);
        float total = 0.0f;
        for (int j = 0; j < n; ++j) {
            const float t = __fsub_rn((float)(j + x0), c);
            const float arg = fabsf((float)(((double)t + 0.5) * (double)invscale));
            w[j] = arg < 1.0f ? __fsub_rn(1.0f, arg) : 0.0f;
            total = __fadd_rn(total, w[j]);
        }
        if (total != 0.0f)
            for (int j = 0; j < n; ++j) w[j] = __fdiv_rn(w[j], total);
    }
};

// One band of one resampled sample: the fp32 tile holds the horizontal pass of source rows [ylo, ylo + srows) of the
// box; value() runs the vertical pass of window pixel (r, x, c) of the band and normalises it.
template <bool kBf16>
struct ResampleBand {
    const float *tile, *wy, *mean, *std;
    const int *ymin, *ysize;
    int ylo, rowf, ky, C, ow, flip, ok;

    __device__ __forceinline__ uint32_t value(int r, int x, int c) const {
        if (!ok) return kBf16 ? 0x7fc0u : 0x7fc00000u;  // a box outside the image: quiet NaN, nothing read
        const int u = flip ? ow - 1 - x : x;
        const float *col = tile + (ymin[r] - ylo) * rowf + u * C + c;
        const float *w = wy + r * ky;
        const int n = ysize[r];
        float acc = __fmul_rn(col[0], w[0]);
        for (int j = 1; j < n; ++j) acc = __fadd_rn(acc, __fmul_rn(col[j * rowf], w[j]));
        const float v = __fdiv_rn(__fsub_rn(acc, mean[c]), std[c]);
        return kBf16 ? (uint32_t)f32_to_bf16(v) : __float_as_uint(v);
    }
};

// Dynamic shared memory of one CTA, in this order (every piece a multiple of 4 bytes).
struct ResampleSmem {
    float *tile, *wx, *wy;
    int *xmin, *xsize, *ymin, *ysize;

    __host__ __device__ static size_t bytes(int srows, int rowf, int ow, int kx, int rows, int ky) {
        return 4 * ((size_t)srows * rowf + (size_t)ow * (kx + 2) + (size_t)rows * (ky + 2));
    }
    __device__ ResampleSmem(float *base, const ResampleArgs &a) {
        tile = base;
        wx = tile + (size_t)a.srows * a.ow * a.C;
        wy = wx + (size_t)a.ow * a.kx;
        xmin = reinterpret_cast<int *>(wy + (size_t)a.rows * a.ky);
        xsize = xmin + a.ow;
        ymin = xsize + a.ow;
        ysize = ymin + a.rows;
    }
};

template <bool kBf16, bool kNHWC>
__global__ void __launch_bounds__(kResampleThreads) image_resample_u8_kernel(const ResampleArgs a) {
    extern __shared__ float s_dyn[];
    __shared__ float s_lut[256];
    __shared__ float s_norm[8];
    const ResampleSmem sm(s_dyn, a);
    for (int e = threadIdx.x; e < 256; e += blockDim.x) s_lut[e] = __fdiv_rn((float)e, 255.0f);
    if (threadIdx.x < 4) {
        s_norm[threadIdx.x] = a.mean[threadIdx.x];
        s_norm[4 + threadIdx.x] = a.std[threadIdx.x];
    }
    const long long jobs = a.batch * a.bands;
    const int rowf = a.ow * a.C, plane = a.oh * a.ow;
    for (long long job = blockIdx.x; job < jobs; job += gridDim.x) {
        const long long i = job / a.bands;
        const int y0 = (int)(job - i * a.bands) * a.rows;
        const int nr = min(a.rows, a.oh - y0);
        const int *box = a.boxes + 5 * i;
        const int top = box[0], left = box[1], bh = box[2], bw = box[3], flip = box[4] != 0;
        const int ok = top >= 0 && left >= 0 && bh >= 1 && bw >= 1 && top <= a.H - bh && left <= a.W - bw;
        const ResampleAxis ax(ok ? bw : 1, a.rw), ay(ok ? bh : 1, a.rh);
        const int ylo = ay.xmin(a.win_top + y0);
        const int nsrc = ok ? min(ay.xend(a.win_top + y0 + nr - 1) - ylo, a.srows) : 0;
        __syncthreads();  // the previous job's readers are done with the tile and the taps (and the tables are built)
        if (ok) {
            for (int u = threadIdx.x; u < a.ow; u += blockDim.x)
                ax.taps(a.win_left + u, sm.xmin[u], sm.xsize[u], sm.wx + u * a.kx);
            for (int r = threadIdx.x; r < nr; r += blockDim.x)
                ay.taps(a.win_top + y0 + r, sm.ymin[r], sm.ysize[r], sm.wy + r * a.ky);
        }
        __syncthreads();
        const uint8_t *img = a.images + a.idx[i] * a.sample_bytes + ((long long)(top + ylo) * a.W + left) * a.C;
        for (int t = threadIdx.x; t < nsrc * rowf; t += blockDim.x) {
            const int sr = t / rowf, e = t - sr * rowf, u = e / a.C, c = e - u * a.C;
            const uint8_t *src = img + ((long long)sr * a.W + sm.xmin[u]) * a.C + c;
            const float *w = sm.wx + u * a.kx;
            const int n = sm.xsize[u];
            float acc = __fmul_rn(s_lut[__ldg(src)], w[0]);
            for (int j = 1; j < n; ++j) acc = __fadd_rn(acc, __fmul_rn(s_lut[__ldg(src + j * a.C)], w[j]));
            sm.tile[t] = acc;
        }
        __syncthreads();
        const ResampleBand<kBf16> band{sm.tile, sm.wy, s_norm, s_norm + 4, sm.ymin, sm.ysize, ylo, rowf, a.ky, a.C,
                                       a.ow, flip, ok};
        if (kNHWC) {
            const int C = a.C, ow = a.ow;
            image_store_run<kBf16>(a.out, i * plane * C + (long long)y0 * ow * C, nr * ow * C, [&](int k) {
                const int p = k / C;
                return ImageCursor<ResampleBand<kBf16>, true>{band, p / ow, p - (p / ow) * ow, k - p * C};
            });
        } else {
            for (int c = 0; c < a.C; ++c) {
                const int ow = a.ow;
                image_store_run<kBf16>(a.out, (i * a.C + c) * plane + (long long)y0 * ow, nr * ow, [&](int k) {
                    return ImageCursor<ResampleBand<kBf16>, false>{band, k / ow, k - (k / ow) * ow, c};
                });
            }
        }
    }
}

// Band geometry of one launch (host): taps per output on each axis at the largest box the image allows, the band
// height whose tile and row taps fit kResampleBandBytes (at least one row), and the tile rows that band can need.
// The column taps take ow (kx + 2) words whatever the band height, so a launch needs at most the column taps plus the
// larger of kResampleBandBytes and a band of one row: kResampleMaxSmem at the widest row and the largest downscale.
struct ResamplePlan {
    int kx, ky, rows, bands, srows;
    size_t smem;
};

static int resample_taps(int in, int out) {
    const float scale = (float)in / (float)out;
    return (int)std::ceil(scale >= 1.0f ? scale : 1.0f) * 2 + 1;
}

// Source rows a band of `rows` output rows can read: (rows - 1) scale + 2 support + 1, plus 2 for rounding.
static int resample_srows(int rows, int H, int rh) {
    const double scale = (double)H / (double)rh, support = scale >= 1.0 ? scale : 1.0;
    const int n = (int)std::floor((rows - 1) * scale + 2.0 * support + 1.0) + 2;
    return n < H ? n : H;
}

constexpr int kResampleMaxTaps = 2 * kResampleMaxScale + 1;
constexpr int kResampleMaxSrows = 2 * kResampleMaxScale + 3;  // resample_srows(1, H, rh) at H = 8 rh
constexpr size_t kResampleMaxSmem = 4 * ((size_t)kResampleMaxRowElems * (kResampleMaxTaps + 2) +
                                         (size_t)kResampleMaxSrows * kResampleMaxRowElems + (kResampleMaxTaps + 2));
static_assert(kResampleMaxSmem > (size_t)kResampleBandBytes, "a band of one row at the limits exceeds the band target");
static_assert(kResampleMaxSmem + 2048 <= 227 * 1024, "every accepted launch must fit the opt-in shared memory of sm_90");

static ResamplePlan resample_plan(int H, int W, int C, int rh, int rw, int oh, int ow) {
    ResamplePlan p;
    p.kx = resample_taps(W, rw);
    p.ky = resample_taps(H, rh);
    const size_t row_bytes = (size_t)ow * C * 4;
    auto band_bytes = [&](int rows) { return 4 * (size_t)rows * (p.ky + 2) + resample_srows(rows, H, rh) * row_bytes; };
    int rows = 1;
    while (rows < oh && band_bytes(rows + 1) <= (size_t)kResampleBandBytes) ++rows;
    p.bands = (oh + rows - 1) / rows;
    p.rows = (oh + p.bands - 1) / p.bands;
    p.srows = resample_srows(p.rows, H, rh);
    p.smem = ResampleSmem::bytes(p.srows, ow * C, ow, p.kx, p.rows, p.ky);
    return p;
}

template <bool kBf16, bool kNHWC>
static int launch_resample(int grid, size_t smem, cudaStream_t st, const ResampleArgs &a) {
    DMLB_CUDA(cudaFuncSetAttribute(image_resample_u8_kernel<kBf16, kNHWC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem));
    image_resample_u8_kernel<kBf16, kNHWC><<<grid, kResampleThreads, smem, st>>>(a);
    return launched();
}

}  // namespace dmlb

using namespace dmlb;

extern "C" {

int dmlb_shard_gather_u8(const uint8_t *images, const int64_t *idx, int64_t batch, int64_t row_elems, float mean,
                         float std, void *out, int out_bf16, void *stream) {
    if (!images || !idx || !out || batch < 0 || row_elems <= 0 || std == 0.0f) return DMLB_EINVAL;
    if (batch == 0) return DMLB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec = (row_elems % 16 == 0) && (((uintptr_t)images & 15) == 0) && (((uintptr_t)out & 15) == 0);
    if (vec) {
        long long vpr = row_elems / 16;
        int grid = grid_for(batch * vpr, 256);
        if (out_bf16)
            shard_gather_u8_kernel<true><<<grid, 256, 0, st>>>(images, (const long long *)idx, batch, row_elems, vpr, mean, std, out);
        else
            shard_gather_u8_kernel<false><<<grid, 256, 0, st>>>(images, (const long long *)idx, batch, row_elems, vpr, mean, std, out);
    } else {
        int grid = grid_for(batch * row_elems, 256);
        if (out_bf16)
            shard_gather_u8_scalar_kernel<true><<<grid, 256, 0, st>>>(images, (const long long *)idx, batch, row_elems, mean, std, out);
        else
            shard_gather_u8_scalar_kernel<false><<<grid, 256, 0, st>>>(images, (const long long *)idx, batch, row_elems, mean, std, out);
    }
    return launched();
}

int dmlb_shard_gather_i64(const int64_t *labels, const int64_t *idx, int64_t batch, int64_t *labels_out, void *stream) {
    if (!labels || !idx || !labels_out || batch < 0) return DMLB_EINVAL;
    if (batch == 0) return DMLB_OK;
    shard_gather_i64_kernel<<<grid_for(batch, 256), 256, 0, (cudaStream_t)stream>>>(
        (const long long *)labels, (const long long *)idx, batch, (long long *)labels_out);
    return launched();
}

int dmlb_shard_slice(const int64_t *perm, int64_t first, int64_t count, int64_t rank, int64_t world, int64_t *idx_out,
                     void *stream) {
    if (!perm || !idx_out || first < 0 || count < 0 || world < 1 || rank < 0 || rank >= world) return DMLB_EINVAL;
    if (count == 0) return DMLB_OK;
    shard_slice_kernel<<<grid_for(count, 256), 256, 0, (cudaStream_t)stream>>>((const long long *)perm, first, count, rank,
                                                                               world, (long long *)idx_out);
    return launched();
}

int dmlb_image_batch_u8(const uint8_t *images, const int64_t *idx, int64_t batch, int32_t H, int32_t W, int32_t C,
                        int32_t out_h, int32_t out_w, int32_t pad, int crop_mode, int hflip, uint64_t seed, int64_t epoch,
                        const dmlb_image_norm *norm, void *out, int out_bf16, int channels_last, int32_t *params_out,
                        void *stream) {
    if (batch < 0 || !norm || C < 1 || C > 4 || H < 1 || W < 1 || out_h < 1 || out_w < 1 || pad < 0) return DMLB_EINVAL;
    if ((crop_mode != 0 && crop_mode != 1) || (long long)out_h > (long long)H + 2LL * pad ||
        (long long)out_w > (long long)W + 2LL * pad)
        return DMLB_EINVAL;
    for (int c = 0; c < C; ++c)
        if (norm->std[c] == 0.0f) return DMLB_EINVAL;
    if (batch > 0 && (!images || !idx || !out)) return DMLB_EINVAL;
    const long long rowcap = ((long long)out_w * C + 15) / 16 * 16 + 16;
    if (rowcap > kImageMaxRowBytes) return DMLB_EINVAL;
    if (((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0) return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    ImageArgs a;
    a.images = images;
    a.idx = (const long long *)idx;
    a.out = out;
    a.params = params_out;
    a.batch = batch;
    a.sample_bytes = (long long)H * W * C;
    a.seed = seed;
    a.epoch = epoch;
    a.H = H, a.W = W, a.C = C, a.oh = out_h, a.ow = out_w, a.pad = pad;
    a.random_crop = crop_mode, a.hflip = hflip ? 1 : 0;
    const int max_rows = (int)(kImageBandBytes / rowcap) > 0 ? (int)(kImageBandBytes / rowcap) : 1;
    a.bands = (out_h + max_rows - 1) / max_rows;
    a.rows = (out_h + a.bands - 1) / a.bands;
    a.rowcap = (int)rowcap;
    for (int c = 0; c < 4; ++c) {
        a.mean[c] = c < C ? norm->mean[c] : 0.0f;
        a.std[c] = c < C ? norm->std[c] : 1.0f;
    }
    const long long jobs = batch * a.bands;
    const long long cap = (long long)sm_count() * kImageCtasPerSm;
    const int grid = (int)(jobs < cap ? jobs : cap);
    const size_t smem = (size_t)a.rows * a.rowcap;
    const bool vec_load = ((uintptr_t)images & 15) == 0;
    cudaStream_t st = (cudaStream_t)stream;
    if (out_bf16) {
        if (channels_last)
            launch_image<true, true>(vec_load, grid, smem, st, a);
        else
            launch_image<true, false>(vec_load, grid, smem, st, a);
    } else {
        if (channels_last)
            launch_image<false, true>(vec_load, grid, smem, st, a);
        else
            launch_image<false, false>(vec_load, grid, smem, st, a);
    }
    return launched();
}


int dmlb_image_resample_u8(const uint8_t *images, const int64_t *idx, const int32_t *boxes, int64_t batch, int32_t H,
                           int32_t W, int32_t C, int32_t resize_h, int32_t resize_w, int32_t win_top, int32_t win_left,
                           int32_t out_h, int32_t out_w, const dmlb_image_norm *norm, void *out, int out_bf16,
                           int channels_last, void *stream) {
    if (batch < 0 || !norm || C < 1 || C > 4) return DMLB_EINVAL;
    for (int32_t side : {H, W, resize_h, resize_w, out_h, out_w})
        if (side < 1 || side > kResampleMaxSide) return DMLB_EINVAL;
    if ((long long)H > (long long)kResampleMaxScale * resize_h || (long long)W > (long long)kResampleMaxScale * resize_w)
        return DMLB_EINVAL;
    if (win_top < 0 || win_left < 0 || win_top > resize_h - out_h || win_left > resize_w - out_w) return DMLB_EINVAL;
    if ((long long)out_w * C > kResampleMaxRowElems) return DMLB_EINVAL;
    for (int c = 0; c < C; ++c)
        if (norm->std[c] == 0.0f) return DMLB_EINVAL;
    if (batch > 0 && (!images || !idx || !boxes || !out)) return DMLB_EINVAL;
    if (((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0 || ((uintptr_t)boxes & 3) != 0) return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    const ResamplePlan p = resample_plan(H, W, C, resize_h, resize_w, out_h, out_w);
    ResampleArgs a;
    a.images = images;
    a.idx = (const long long *)idx;
    a.boxes = boxes;
    a.out = out;
    a.batch = batch;
    a.sample_bytes = (long long)H * W * C;
    a.H = H, a.W = W, a.C = C, a.rh = resize_h, a.rw = resize_w, a.win_top = win_top, a.win_left = win_left;
    a.oh = out_h, a.ow = out_w;
    a.rows = p.rows, a.bands = p.bands, a.srows = p.srows, a.kx = p.kx, a.ky = p.ky;
    for (int c = 0; c < 4; ++c) {
        a.mean[c] = c < C ? norm->mean[c] : 0.0f;
        a.std[c] = c < C ? norm->std[c] : 1.0f;
    }
    const long long jobs = batch * p.bands;
    const long long cap = (long long)sm_count() * kResampleCtasPerSm;
    const int grid = (int)(jobs < cap ? jobs : cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (out_bf16)
        return channels_last ? launch_resample<true, true>(grid, p.smem, st, a)
                             : launch_resample<true, false>(grid, p.smem, st, a);
    return channels_last ? launch_resample<false, true>(grid, p.smem, st, a)
                         : launch_resample<false, false>(grid, p.smem, st, a);
}

}  // extern "C"
