// Device-resident data-shard iterator kernels (SURVEY §8f-1).
//
// Reference: util/data.py:11-30 shard_indices (`indices[rank::world]` after the optional MT19937 shuffle and tail drop)
// and examples/mnist.py:16-21 (torchvision ToTensor + Normalize((0.1307,), (0.3081,)) + DataLoader batching, on the host).
// Here the whole uint8 dataset stays in HBM (MNIST: 47 MB of 180 GB); the epoch permutation is uploaded once per epoch
// (bit-exact host computation — the same numpy MT19937 stream the reference uses) and each step is one gather kernel:
//   out[i, :] = (float(images[idx[i], :]) / 255 - mean) / std                      784 B read, 3136 (fp32) B written / sample
// HBM-bound byte work: 16 pixels (one 128-bit load) per thread, 4x 128-bit stores, rows found through idx[] (L2-resident).
#include <cmath>
#include <type_traits>

#include <cooperative_groups.h>

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
// (include/dmlb.h states the rule.)  One CTA job = one band of up to `rows` output rows of one sample, at the window
// {top, left, flipped} the host gave it in `windows`.  The band's window rows are staged into shared memory
// as the 16-byte aligned chunks of the source rows that cover them (so the loads are 128-bit whatever the crop offset),
// then written out in the output's contiguous order, 16-byte stores for the body of every contiguous run.  Normalised
// values come from a per-launch [C][256] table in shared memory built with norm_px, so every element is two shared
// loads and no division.  HBM traffic is the window bytes (plus < 32 B of chunk rounding per row) and the output.

constexpr int kImageThreads = 256;
constexpr int kImageBandBytes = 24576;  // staged window bytes per CTA (+ the 4 KB table)
constexpr int kImageCtasPerSm = 6;      // grid cap: what fits one SM at <= 40 registers (__launch_bounds__ holds it)
constexpr int kImageMaxRowBytes = 49152;

struct ImageArgs {
    const uint8_t *images;
    const long long *idx;
    const int *windows;
    void *out;
    long long batch, sample_bytes;
    int H, W, C, oh, ow, pad;
    long long dy, dx;         // a window's top lies in [0, dy], its left in [0, dx] (H + 2 pad may pass INT_MAX)
    int rows, bands, rowcap;  // band height, bands per sample, staged bytes per window row
    float mean[4], std[4];
};

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
// Band: any band type with members C, ow and value(r, x, c) (ImageBand, NanBand, ResampleBand).
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

// Rows [y0, y0 + nr) of sample i of the logical [batch, C, oh, ow] output a.out (plane = oh * ow), written in its
// memory order (NCHW: one run per channel plane, NHWC: one run) from band.value.  Args: ImageArgs or ResampleArgs.
template <bool kBf16, bool kNHWC, class Args, class Band>
__device__ __forceinline__ void store_band(const Args &a, long long i, int y0, int nr, int plane, const Band &band) {
    if (kNHWC) {
        const int C = a.C, ow = a.ow;
        image_store_run<kBf16>(a.out, i * plane * C + (long long)y0 * ow * C, nr * ow * C, [&](int k) {
            const int p = k / C;
            return ImageCursor<Band, true>{band, p / ow, p - (p / ow) * ow, k - p * C};
        });
    } else {
        for (int c = 0; c < a.C; ++c) {
            const int ow = a.ow;
            image_store_run<kBf16>(a.out, (i * a.C + c) * plane + (long long)y0 * ow, nr * ow, [&](int k) {
                return ImageCursor<Band, false>{band, k / ow, k - (k / ow) * ow, c};
            });
        }
    }
}

// The band of a sample whose window lies outside the padded image: quiet NaN, nothing read.
template <bool kBf16>
struct NanBand {
    int C, ow;
    __device__ __forceinline__ uint32_t value(int, int, int) const { return kBf16 ? 0x7fc0u : 0x7fc00000u; }
};

template <bool kBf16, bool kNHWC, bool kVecLoad>
__global__ void __launch_bounds__(kImageThreads, kImageCtasPerSm) image_batch_u8_kernel(const ImageArgs a) {
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
        const int top = a.windows[3 * i], left = a.windows[3 * i + 1], flip = a.windows[3 * i + 2] != 0;
        if (top < 0 || top > a.dy || left < 0 || left > a.dx) {
            store_band<kBf16, kNHWC>(a, i, y0, nr, plane, NanBand<kBf16>{a.C, a.ow});
            continue;
        }
        const long long row = a.idx[i];
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
        store_band<kBf16, kNHWC>(a, i, y0, nr, plane,
                                 ImageBand<kVecLoad>{sm, s_lut, (uint32_t)(uintptr_t)col0, sy0, a.H, WC, a.C, a.ow,
                                                     u_lo, u_hi, a.rowcap, flip});
    }
}

template <bool kBf16, bool kNHWC>
static int launch_image(bool vec_load, int grid, size_t smem, cudaStream_t st, const ImageArgs &a) {
    if (vec_load)
        image_batch_u8_kernel<kBf16, kNHWC, true><<<grid, kImageThreads, smem, st>>>(a);
    else
        image_batch_u8_kernel<kBf16, kNHWC, false><<<grid, kImageThreads, smem, st>>>(a);
    return launched();
}

// ---- host scaffolding of the two band kernels -----------------------------------------------------------------------

// Refuses std[c] == 0 for c < C; otherwise fills the kernel's 4-channel mean and std (channels past C: 0 and 1).
static bool pack_norm(const dmlb_image_norm *norm, int C, float *mean, float *std) {
    for (int c = 0; c < C; ++c)
        if (norm->std[c] == 0.0f) return false;
    for (int c = 0; c < 4; ++c) {
        mean[c] = c < C ? norm->mean[c] : 0.0f;
        std[c] = c < C ? norm->std[c] : 1.0f;
    }
    return true;
}

// One CTA per band job, at most ctas_per_sm CTAs per SM (each CTA then walks several jobs).
static int band_grid(long long jobs, int ctas_per_sm) {
    const long long cap = (long long)sm_count() * ctas_per_sm;
    return (int)(jobs < cap ? jobs : cap);
}

// Returns launch(bf16, nhwc), the two passed as std::bool_constant so that launch can name a kernel instance.
template <class Launch>
static int dispatch_layout(int out_bf16, int channels_last, const Launch &launch) {
    using T = std::true_type;
    using F = std::false_type;
    if (out_bf16) return channels_last ? launch(T{}, T{}) : launch(T{}, F{});
    return channels_last ? launch(F{}, T{}) : launch(F{}, F{});
}


// ---- resampled colour images: box -> antialiased bilinear resize -> window -> flip -> normalise ---------------------
// (dmlb_image_resample_u8 and, over images of different sizes, dmlb_image_resample_ragged_u8; include/dmlb.h states
// the rule.)  One CTA job = one band of up to `rows` output rows of one sample.  The CTA builds the sample's column taps (xmin, xsize, weights) for the window's columns and the row taps of
// the band, runs the horizontal pass over the band's source rows into an fp32 [srows][out_w * C] tile in shared memory,
// then the vertical pass, written in the output's contiguous order by store_band.  Source bytes are read through
// L1 (a box row's bytes are read by neighbouring columns' taps) and mapped through a 256-entry fl32(byte) / 255 table.
// Every operation of the tap and pixel arithmetic is rounded once, as written (no FMA contraction).

constexpr int kResampleThreads = 256;
constexpr int kResampleMaxScale = 8;          // H <= 8 resize_h, W <= 8 resize_w: at most 2 * 8 + 1 taps per output
constexpr int kResampleMaxRowElems = 1024;    // out_w * C
constexpr int kResampleMaxSide = 32768;       // H, W, resize_h, resize_w: tap positions stay exact in fp32
constexpr int kResampleBandBytes = 32768;     // target size of a band's tile + row taps (one row may need up to 76 KB)
constexpr int kResampleCtasPerSm = 4;

struct ResampleArgs {
    const uint8_t *images;              // [n, H, W, C] images (LaunchGeometry) or the packed store (TableGeometry)
    const long long *idx;
    const int *geom;                    // boxes [batch][5] (LaunchGeometry) or geometry rows [batch][9] (TableGeometry)
    const dmlb_image_extent *extents;   // TableGeometry: one row per image of the store
    void *out;
    long long batch, sample_bytes;      // sample_bytes: H W C (LaunchGeometry) or the store's bytes (TableGeometry)
    int H, W, C, rh, rw, win_top, win_left, oh, ow;  // H .. win_left: LaunchGeometry only
    int rows, bands, srows, kx, ky;  // band height, bands per sample, tile rows, column / row tap stride
    float mean[4], std[4];
};

// One sample's geometry: its image (H x W; where it starts is Geometry::image's), box, flip, resized size and window.
struct ResampleSample {
    long long offset;  // TableGeometry: the image's byte offset into the store
    int H, W, top, left, bh, bw, flip, rh, rw, win_top, win_left;
};

__host__ __device__ __forceinline__ double resample_dmul(double x, double y) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(x, y);
#else
    return x * y;
#endif
}
__host__ __device__ __forceinline__ double resample_dadd(double x, double y) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(x, y);
#else
    return x + y;
#endif
}

// Source rows a band of `rows` output rows can read when `in` rows resize to `out`: (rows - 1) scale + 2 support + 1,
// plus 2 for the fp32 rounding of the tap centres (their error stays below 0.01 row at sides of 32768).  The host
// plans with it and the kernel admits samples with it, both rounding every operation once, so they agree bit for bit.
__host__ __device__ __forceinline__ int resample_band_rows(int rows, int in, int out) {
    const double scale = (double)in / (double)out, support = scale >= 1.0 ? scale : 1.0;
    return (int)floor(resample_dadd(resample_dadd(resample_dmul(rows - 1, scale), 2.0 * support), 1.0)) + 2;
}

// Where a sample's geometry comes from.  LaunchGeometry (dmlb_image_resample_u8): the image size, resized size and
// window are launch constants the host has checked, the box is row i of a [batch][5] table.  TableGeometry
// (dmlb_image_resample_ragged_u8): the image's extent row and row i of a [batch][9] table, both unchecked device data;
// a sample whose extent lies outside the store or whose window lies outside its resized image comes back with an empty
// box (and a 1 x 1 resize), which the kernel's box check turns into a NaN sample.
struct LaunchGeometry {
    __device__ __forceinline__ static ResampleSample at(const ResampleArgs &a, long long i) {
        const int *g = a.geom + 5 * i;
        return {0, a.H, a.W, g[0], g[1], g[2], g[3], g[4] != 0, a.rh, a.rw, a.win_top, a.win_left};
    }
    __device__ __forceinline__ static const uint8_t *image(const ResampleArgs &a, long long i, const ResampleSample &) {
        return a.images + a.idx[i] * a.sample_bytes;
    }
    // The plan is the image's own: every box inside the image fits it.
    __device__ __forceinline__ static bool fits(const ResampleArgs &, const ResampleSample &, int, int) { return true; }
};

struct TableGeometry {
    __device__ __forceinline__ static ResampleSample at(const ResampleArgs &a, long long i) {
        const int *g = a.geom + 9 * i;
        const dmlb_image_extent e = a.extents[a.idx[i]];
        const int rh = g[5], rw = g[6], wt = g[7], wl = g[8];
        const bool valid = e.H >= 1 && e.W >= 1 && e.H <= kResampleMaxSide && e.W <= kResampleMaxSide &&
                           e.offset >= 0 && e.offset <= a.sample_bytes - (long long)e.H * e.W * a.C && rh >= 1 &&
                           rw >= 1 && rh <= kResampleMaxSide && rw <= kResampleMaxSide && wt >= 0 && wl >= 0 &&
                           wt <= rh - a.oh && wl <= rw - a.ow;
        if (!valid) return {0, 1, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0};
        return {e.offset, e.H, e.W, g[0], g[1], g[2], g[3], g[4] != 0, rh, rw, wt, wl};
    }
    __device__ __forceinline__ static const uint8_t *image(const ResampleArgs &a, long long, const ResampleSample &s) {
        return a.images + s.offset;
    }
    // The plan is the launch bounds': taps within the strides, a band's source rows within the tile.
    __device__ __forceinline__ static bool fits(const ResampleArgs &a, const ResampleSample &s, int kx, int ky) {
        return kx <= a.kx && ky <= a.ky && min(resample_band_rows(a.rows, s.bh, s.rh), s.bh) <= a.srows;
    }
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

// A sample is admitted when its box lies inside its image and it fits the launch's plan in every band job
// (Geometry::fits: taps per output within the strides kx, ky and a band's source rows within the tile, by
// resample_band_rows at the launch's band height or the box height when that is less).  The test depends on the
// sample alone, so every band job of a sample decides alike: an admitted sample is resampled whole, any other reads
// nothing and is quiet NaN whole.
template <bool kBf16, bool kNHWC, class Geometry>
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
        const ResampleSample s = Geometry::at(a, i);
        int ok = s.top >= 0 && s.left >= 0 && s.bh >= 1 && s.bw >= 1 && s.top <= s.H - s.bh && s.left <= s.W - s.bw;
        const ResampleAxis ax(ok ? s.bw : 1, s.rw), ay(ok ? s.bh : 1, s.rh);
        ok = ok && Geometry::fits(a, s, ax.K, ay.K);
        const int flip = s.flip;
        const int ylo = ay.xmin(s.win_top + y0);
        const int nsrc = ok ? ay.xend(s.win_top + y0 + nr - 1) - ylo : 0;
        __syncthreads();  // the previous job's readers are done with the tile and the taps (and the tables are built)
        if (ok) {
            for (int u = threadIdx.x; u < a.ow; u += blockDim.x)
                ax.taps(s.win_left + u, sm.xmin[u], sm.xsize[u], sm.wx + u * a.kx);
            for (int r = threadIdx.x; r < nr; r += blockDim.x)
                ay.taps(s.win_top + y0 + r, sm.ymin[r], sm.ysize[r], sm.wy + r * a.ky);
        }
        __syncthreads();
        const uint8_t *img = Geometry::image(a, i, s) + ((long long)(s.top + ylo) * s.W + s.left) * a.C;
        for (int t = threadIdx.x; t < nsrc * rowf; t += blockDim.x) {
            const int sr = t / rowf, e = t - sr * rowf, u = e / a.C, c = e - u * a.C;
            const uint8_t *src = img + ((long long)sr * s.W + sm.xmin[u]) * a.C + c;
            const float *w = sm.wx + u * a.kx;
            const int n = sm.xsize[u];
            float acc = __fmul_rn(s_lut[__ldg(src)], w[0]);
            for (int j = 1; j < n; ++j) acc = __fadd_rn(acc, __fmul_rn(s_lut[__ldg(src + j * a.C)], w[j]));
            sm.tile[t] = acc;
        }
        __syncthreads();
        store_band<kBf16, kNHWC>(a, i, y0, nr, plane,
                                 ResampleBand<kBf16>{sm.tile, sm.wy, s_norm, s_norm + 4, sm.ymin, sm.ysize, ylo, rowf,
                                                     a.ky, a.C, a.ow, flip, ok});
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

// Tile rows of a band of `rows` output rows: resample_band_rows, capped by the most rows a box can have.
static int resample_srows(int rows, int H, int rh, int max_box_h) {
    const int n = resample_band_rows(rows, H, rh);
    return n < max_box_h ? n : max_box_h;
}

constexpr int kResampleMaxTaps = 2 * kResampleMaxScale + 1;
constexpr int kResampleMaxSrows = 2 * kResampleMaxScale + 3;  // resample_srows(1, H, rh) at H = 8 rh
constexpr size_t kResampleMaxSmem = 4 * ((size_t)kResampleMaxRowElems * (kResampleMaxTaps + 2) +
                                         (size_t)kResampleMaxSrows * kResampleMaxRowElems + (kResampleMaxTaps + 2));
static_assert(kResampleMaxSmem > (size_t)kResampleBandBytes, "a band of one row at the limits exceeds the band target");
static_assert(kResampleMaxSmem + 2048 <= 227 * 1024, "every accepted launch must fit the opt-in shared memory of sm_90");

// The plan of boxes of up to H x W resized to rh x rw, boxes at most max_box_h rows high (H for one image size; the
// largest side the kernel takes when the launch bounds only the downscale).
static ResamplePlan resample_plan(int H, int W, int C, int rh, int rw, int oh, int ow, int max_box_h) {
    ResamplePlan p;
    p.kx = resample_taps(W, rw);
    p.ky = resample_taps(H, rh);
    const size_t row_bytes = (size_t)ow * C * 4;
    auto band_bytes = [&](int rows) {
        return 4 * (size_t)rows * (p.ky + 2) + resample_srows(rows, H, rh, max_box_h) * row_bytes;
    };
    int rows = 1;
    while (rows < oh && band_bytes(rows + 1) <= (size_t)kResampleBandBytes) ++rows;
    p.bands = (oh + rows - 1) / rows;
    p.rows = (oh + p.bands - 1) / p.bands;
    p.srows = resample_srows(p.rows, H, rh, max_box_h);
    p.smem = ResampleSmem::bytes(p.srows, ow * C, ow, p.kx, p.rows, p.ky);
    return p;
}

template <bool kBf16, bool kNHWC, class Geometry>
static int launch_resample(int grid, size_t smem, cudaStream_t st, const ResampleArgs &a) {
    DMLB_CUDA(cudaFuncSetAttribute(image_resample_u8_kernel<kBf16, kNHWC, Geometry>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    image_resample_u8_kernel<kBf16, kNHWC, Geometry><<<grid, kResampleThreads, smem, st>>>(a);
    return launched();
}

// The launch both resample entries share, on arguments they have checked.  a.images, a.idx, a.geom, a.extents,
// a.sample_bytes, the LaunchGeometry fields and the norm are the caller's.
template <class Geometry>
static int resample_launch(ResampleArgs &a, const ResamplePlan &p, int64_t batch, int32_t C, int32_t out_h,
                           int32_t out_w, void *out, int out_bf16, int channels_last, void *stream) {
    a.out = out;
    a.batch = batch;
    a.C = C, a.oh = out_h, a.ow = out_w;
    a.rows = p.rows, a.bands = p.bands, a.srows = p.srows, a.kx = p.kx, a.ky = p.ky;
    const int grid = band_grid(batch * p.bands, kResampleCtasPerSm);
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_layout(out_bf16, channels_last, [&](auto bf16, auto nhwc) {
        return launch_resample<decltype(bf16)::value, decltype(nhwc)::value, Geometry>(grid, p.smem, st, a);
    });
}

// ---- batch mixing: random erasing -> MixUp or CutMix -> soft targets (dmlb_image_mix) --------------------------------
// (include/dmlb.h states the rule.)  Thread t owns V consecutive elements of a sample (one 16-byte output store: 4 fp32
// or 8 bf16 values; V = 1 when a sample's elements or the pointers are not 16-byte aligned) and walks a segment of the
// batch in order, keeping the previous sample's erased values in registers: the fp32 scratch batch is read once, plus
// the partner of each segment's first sample, and `out` is written once.  The segments of one position are spread over
// blockIdx.y so that a small batch still fills the GPU.  The targets are written by the same threads afterwards.

constexpr int kMixThreads = 256;
constexpr int kMixUnroll = 4;       // samples loaded ahead of their stores
constexpr int kMixCtasPerSm = 8;    // target grid: enough segments to put this many CTAs on every SM
constexpr int kMixMaxSide = 32768;  // h, w

struct MixArgs {
    const float *src;
    const long long *idx, *labels;
    const int *erase;
    void *out, *targets;
    long long batch, S;        // samples, elements per sample
    long long nvec;            // positions per sample (S / V)
    int seglen, h, w, C, nhwc, mode, y1, y2, x1, x2, K;
    float w_prev, w_cur;       // fl32(1 - lam), fl32(lam)
    float fill[4];
};

// The erase box of sample j: on, and whether it is valid (include/dmlb.h: an invalid box makes the sample NaN).
struct EraseBox {
    int top, left, bh, bw, on, bad;
    __device__ __forceinline__ EraseBox(const MixArgs &a, long long j) {
        top = left = bh = bw = on = bad = 0;
        if (a.erase) {
            const int *e = a.erase + 5 * j;
            top = __ldg(e), left = __ldg(e + 1), bh = __ldg(e + 2), bw = __ldg(e + 3), on = __ldg(e + 4) != 0;
            bad = on && !(top >= 0 && left >= 0 && bh >= 0 && bw >= 0 && top <= a.h - bh && left <= a.w - bw);
        }
    }
    __device__ __forceinline__ bool covers(int y, int x) const {
        return on && (unsigned)(y - top) < (unsigned)bh && (unsigned)(x - left) < (unsigned)bw;
    }
};

template <int V>
__device__ __forceinline__ void mix_load(const float *p, float *v) {
    if constexpr (V == 1) {
        v[0] = __ldg(p);
    } else {
#pragma unroll
        for (int q = 0; q < V / 4; ++q) {
            const uint4 u = ld_stream_u4(reinterpret_cast<const uint4 *>(p) + q);
            v[4 * q] = __uint_as_float(u.x), v[4 * q + 1] = __uint_as_float(u.y);
            v[4 * q + 2] = __uint_as_float(u.z), v[4 * q + 3] = __uint_as_float(u.w);
        }
    }
}

template <bool kBf16, int V>
__device__ __forceinline__ void mix_store(void *out, long long e, const float *v) {
    if constexpr (V == 1) {
        if (kBf16)
            reinterpret_cast<uint16_t *>(out)[e] = f32_to_bf16(v[0]);
        else
            reinterpret_cast<float *>(out)[e] = v[0];
    } else if constexpr (kBf16) {
        static_assert(V == 8, "bf16 stores take 8 values");
        *reinterpret_cast<uint4 *>(reinterpret_cast<uint16_t *>(out) + e) =
            make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
    } else {
        static_assert(V == 4, "fp32 stores take 4 values");
        *reinterpret_cast<float4 *>(reinterpret_cast<float *>(out) + e) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

template <bool kBf16, int V>
__global__ void __launch_bounds__(kMixThreads) image_mix_kernel(const MixArgs a) {
    const long long pos = (long long)blockIdx.x * kMixThreads + threadIdx.x;
    const long long B = a.batch;
    if (pos < a.nvec) {
        const long long p0 = pos * V;
        // (y, x) and the fill of each owned element: fixed for the whole walk
        int ys[V], xs[V];
        float fv[V];
        uint32_t cut = 0;  // bit k: element k lies in the CutMix box
#pragma unroll
        for (int k = 0; k < V; ++k) {
            const long long p = p0 + k;
            int c, pix;
            if (a.nhwc) {
                pix = (int)(p / a.C), c = (int)(p - (long long)pix * a.C);
            } else {
                const int plane = a.h * a.w;
                c = (int)(p / plane), pix = (int)(p - (long long)c * plane);
            }
            ys[k] = pix / a.w, xs[k] = pix - ys[k] * a.w;
            fv[k] = a.fill[c];
            if (ys[k] >= a.y1 && ys[k] < a.y2 && xs[k] >= a.x1 && xs[k] < a.x2) cut |= 1u << k;
        }
        // the erased values of sample j, and whether they are NaN (an invalid erase box)
        auto erased = [&](long long j, float *v) {
            mix_load<V>(a.src + j * a.S + p0, v);
            const EraseBox box(a, j);
#pragma unroll
            for (int k = 0; k < V; ++k)
                if (box.covers(ys[k], xs[k])) v[k] = fv[k];
            return box.bad;
        };
        const long long i0 = (long long)blockIdx.y * a.seglen;
        const long long i1 = min(i0 + (long long)a.seglen, B);
        float prev[V];
        int prev_bad = 0;
        if (a.mode != 0 && i0 < i1) prev_bad = erased(i0 == 0 ? B - 1 : i0 - 1, prev);
        for (long long i = i0; i < i1; i += kMixUnroll) {
            float cur[kMixUnroll][V];
            int bad[kMixUnroll];
#pragma unroll
            for (int u = 0; u < kMixUnroll; ++u)
                if (i + u < i1) bad[u] = erased(i + u, cur[u]);
#pragma unroll
            for (int u = 0; u < kMixUnroll; ++u) {
                if (i + u >= i1) break;
                float o[V];
#pragma unroll
                for (int k = 0; k < V; ++k) {
                    bool nan = bad[u];
                    if (a.mode == 1) {
                        o[k] = __fadd_rn(__fmul_rn(prev[k], a.w_prev), __fmul_rn(cur[u][k], a.w_cur));
                        nan = nan || prev_bad;
                    } else if (a.mode == 2 && ((cut >> k) & 1u)) {
                        o[k] = prev[k];
                        nan = prev_bad;
                    } else {
                        o[k] = cur[u][k];
                    }
                    if (nan) o[k] = __uint_as_float(0x7fc00000u);
                }
                mix_store<kBf16, V>(a.out, (i + u) * a.S + p0, o);
#pragma unroll
                for (int k = 0; k < V; ++k) prev[k] = cur[u][k];
                prev_bad = bad[u];
            }
        }
    }
    // the targets: int64 labels (mode 0) or soft targets [B][K]
    const long long nthreads = (long long)gridDim.x * gridDim.y * kMixThreads;
    const long long t0 = ((long long)blockIdx.y * gridDim.x + blockIdx.x) * kMixThreads + threadIdx.x;
    if (a.mode == 0) {
        for (long long i = t0; i < B; i += nthreads)
            reinterpret_cast<long long *>(a.targets)[i] = a.labels[a.idx[i]];
        return;
    }
    auto soft = [&](long long e) {
        const long long i = e / a.K;
        const long long k = e - i * a.K;
        const long long cur = a.labels[a.idx[i]], prv = a.labels[a.idx[i == 0 ? B - 1 : i - 1]];
        if (cur < 0 || cur >= a.K || prv < 0 || prv >= a.K) return __uint_as_float(0x7fc00000u);
        return __fadd_rn(__fmul_rn(prv == k ? 1.0f : 0.0f, a.w_prev), __fmul_rn(cur == k ? 1.0f : 0.0f, a.w_cur));
    };
    float *t = reinterpret_cast<float *>(a.targets);
    const long long n = B * a.K;
    const long long head = min(n, (long long)(((16u - ((uint32_t)(uintptr_t)t & 15u)) & 15u) / 4));
    const long long nv = (n - head) / 4, tail0 = head + 4 * nv;
    for (long long q = t0; q < nv; q += nthreads) {
        const long long e = head + 4 * q;
        *reinterpret_cast<float4 *>(t + e) = make_float4(soft(e), soft(e + 1), soft(e + 2), soft(e + 3));
    }
    for (long long q = t0; q < head + (n - tail0); q += nthreads) {
        const long long e = q < head ? q : tail0 + (q - head);
        t[e] = soft(e);
    }
}

template <bool kBf16, int V>
static int launch_mix(dim3 grid, cudaStream_t st, const MixArgs &a) {
    image_mix_kernel<kBf16, V><<<grid, kMixThreads, 0, st>>>(a);
    return launched();
}

// ---- Op chains: TrivialAugmentWide, RandAugment, AutoAugment, then normalise (dmlb_image_trivial_augment, ------------
// dmlb_image_auto_augment; include/dmlb.h states the rule).  One thread-block cluster per sample; CTA r of a cluster
// of n writes elements [r S / n, (r + 1) S / n) of each of the sample's outputs in memory order (image_store_run).
// Contrast, AutoContrast and Equalize first reduce their statistics over pixels [r P / n, (r + 1) P / n) into the
// CTA's shared memory (a 128-bit integer sum, per-channel min / max, per-channel 256-bin histograms), then every CTA
// folds the cluster's partials in rank order through distributed shared memory between two cluster.sync(): exact
// integer and min / max folds, so the result does not depend on the launch geometry.  Every CTA of a cluster holds the
// same sample and the same op chain, so every branch on the op and every cluster.sync() is uniform.  Geometric ops and
// Sharpness gather from the sample, which sits in L2 at these sizes.  A chain's slots but the last write their fp32
// result into a work buffer (ping-pong between two when there are three or more), and the next slot reads it after a
// cluster.sync(); an Identity slot is skipped, so the sample stays in its current buffer.

namespace cg = cooperative_groups;

constexpr int kTaThreads = 256;
constexpr int kTaWarps = kTaThreads / 32;
constexpr int kTaMaxCluster = 8;              // the portable cluster size
constexpr int kTaPixelsPerCta = 4096;         // cluster size = ceil(h w / this), at most kTaMaxCluster
constexpr int kTaMaxSide = 32768;             // h, w
constexpr long long kTaMaxPixels = 1LL << 24; // h w: C h w fits an int run, the contrast sum fits 120 bits
constexpr long long kTaMaxBatch = (1LL << 31) / kTaMaxCluster - 1;  // the grid is batch * cluster CTAs
constexpr int kTaMaxChain = 4;                // ops per sample of dmlb_image_auto_augment
enum { kTaIdentity, kTaShearX, kTaShearY, kTaTranslateX, kTaTranslateY, kTaRotate, kTaBrightness, kTaColor,
       kTaContrast, kTaSharpness, kTaPosterize, kTaSolarize, kTaAutoContrast, kTaEqualize, kTaOps, kTaInvert = kTaOps };

struct TaArgs {
    const float *src;
    float *work;  // min(n_ops - 1, 2) fp32 batches: the results of a chain's inner slots (NULL when n_ops == 1)
    const int *ops;
    void *out;
    long long S, batch;  // S = C h w
    int n_ops, n_codes;  // ops per sample; op codes below n_codes are valid (14: TrivialAugment's, 15: with Invert)
    int C, h, w, nhwc, bilinear;
    float mean[4], std[4];
};

struct TaShared {
    unsigned int hist[3][256];  // this CTA's histograms (read by the cluster)
    unsigned int total[3][256]; // the cluster's
    float lut[3][256];          // Equalize: fp32 output of every uint8 level
    __int128 wsum[kTaWarps];
    float wmin[kTaWarps][3], wmax[kTaWarps][3];
    __int128 sum;               // this CTA's contrast sum
    float mn[3], mx[3];         // this CTA's min / max
    float cmin[3], cinv[3];     // AutoContrast: the subtrahend and divisor of every channel
    float mean;                 // Contrast: the mean gray
};
static_assert(sizeof(TaShared) <= 227 * 1024, "the TrivialAugment CTA must fit the opt-in shared memory of sm_90");

// trunc(f) as a 128-bit integer, exact for |f| < 2^127.
__device__ __forceinline__ __int128 f32_trunc_i128(float f) {
    if (fabsf(f) < 9.223372036854775808e18f) return (__int128)__float2ll_rz(f);
    const uint32_t b = __float_as_uint(f);
    const __int128 m = (__int128)((b & 0x7fffffu) | 0x800000u) << ((int)((b >> 23) & 0xffu) - 150);
    return (b >> 31) ? -m : m;
}

// The fp64 RNE rounding of v.
__device__ __forceinline__ double i128_to_f64(__int128 v) {
    const bool neg = v < 0;
    const unsigned __int128 u = neg ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
    const unsigned long long hi = (unsigned long long)(u >> 64);
    if (hi == 0) return neg ? -__ull2double_rn((unsigned long long)u) : __ull2double_rn((unsigned long long)u);
    const int n = 64 - __clzll((long long)hi);  // u has 64 + n bits: keep the top 64, the rest as a sticky bit
    const unsigned long long top = (unsigned long long)(u >> n) | (unsigned long long)((u << (128 - n)) != 0);
    const double d = ldexp(__ull2double_rn(top), n);
    return neg ? -d : d;
}

__device__ __forceinline__ float ta_clamp01(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }

// to_dtype(uint8) of torchvision: trunc(v * fl32(255.999)), clamped to [0, 255] (NaN -> 0)
__device__ __forceinline__ int ta_quantize(float v) {
    const float t = __fmul_rn(v, (float)255.999);
    return t >= 255.0f ? 255 : (t > 0.0f ? (int)t : 0);
}

// One op of one sample: the op's constants, value(e) of output element e.  src is the sample's current buffer.
// kWork: src is a work buffer that other CTAs of this cluster wrote earlier in this launch.  The non-coherent path
// (__ldg, ld.global.nc) may serve such a read from a cache line filled before the write, so work is read through L2
// (__ldcg), after the cluster.sync() whose release / acquire orders the writes before the reads.  The caller's src is
// read-only for the whole launch (it overlaps neither work nor out), so it keeps the non-coherent path.
template <bool kWork>
struct TaSample {
    const float *src;
    const TaShared *s;
    const float *mean, *std;
    int op, C, h, w, P, nhwc, bilinear, nan, rot;  // rot: 0 none, else rot90 k = rot (4 = identity)
    float mag, f_mul, f_alpha, r[6];

    __device__ __forceinline__ float in(int c, int y, int x) const {
        const int p = y * w + x;
        const float *q = src + (nhwc ? (long long)p * C + c : (long long)c * P + p);
        if constexpr (kWork) return __ldcg(q);
        return __ldg(q);
    }
    __device__ __forceinline__ float tap(int c, int y, int x) const {
        return (unsigned)y < (unsigned)h && (unsigned)x < (unsigned)w ? in(c, y, x) : 0.0f;
    }
    __device__ __forceinline__ float gray(int y, int x) const {  // ATen fuses the two add_(alpha=) into FMAs
        if (C == 1) return in(0, y, x);
        const float l = __fmul_rn(in(0, y, x), (float)0.2989);
        return __fmaf_rn(in(2, y, x), (float)0.114, __fmaf_rn(in(1, y, x), (float)0.587, l));
    }
    __device__ float geometric(int c, int y, int x) const {
        if (rot) {
            if (rot == 1) return in(c, x, w - 1 - y);
            if (rot == 2) return in(c, h - 1 - y, w - 1 - x);
            if (rot == 3) return in(c, h - 1 - x, y);
            return in(c, y, x);
        }
        const float bx = (float)x - 0.5f * (float)(w - 1), by = (float)y - 0.5f * (float)(h - 1);
        const float gx = __fadd_rn(__fmaf_rn(by, r[1], __fmul_rn(bx, r[0])), r[2]);
        const float gy = __fadd_rn(__fmaf_rn(by, r[4], __fmul_rn(bx, r[3])), r[5]);
        const float ix = __fsub_rn(__fmul_rn(__fadd_rn(gx, 1.0f), 0.5f * (float)w), 0.5f);
        const float iy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 1.0f), 0.5f * (float)h), 0.5f);
        if (!bilinear) {
            const float fx = rintf(ix), fy = rintf(iy);
            return fx >= 0.0f && fx < (float)w && fy >= 0.0f && fy < (float)h ? in(c, (int)fy, (int)fx) : 0.0f;
        }
        const float x0 = floorf(ix), y0 = floorf(iy);
        if (!(x0 >= -1.0f && x0 < (float)w && y0 >= -1.0f && y0 < (float)h)) return 0.0f;  // every tap outside
        const float dx = __fsub_rn(ix, x0), dy = __fsub_rn(iy, y0);
        const float ex = __fsub_rn(1.0f, dx), sy = __fsub_rn(1.0f, dy);
        const int xi = (int)x0, yi = (int)y0;
        float v = __fmul_rn(tap(c, yi, xi), __fmul_rn(sy, ex));
        v = __fadd_rn(v, __fmul_rn(tap(c, yi, xi + 1), __fmul_rn(sy, dx)));
        v = __fadd_rn(v, __fmul_rn(tap(c, yi + 1, xi), __fmul_rn(dy, ex)));
        return __fadd_rn(v, __fmul_rn(tap(c, yi + 1, xi + 1), __fmul_rn(dy, dx)));
    }
    __device__ float sharpen(int c, int y, int x) const {
        const float v = in(c, y, x);
        if (h <= 2 || w <= 2) return v;
        if (y == 0 || x == 0 || y == h - 1 || x == w - 1) return ta_clamp01(v);
        const float a = (float)(1.0 / 13.0), b = (float)(5.0 / 13.0);
        float acc = __fmul_rn(in(c, y - 1, x - 1), a);
#pragma unroll
        for (int k = 1; k < 9; ++k) {
            const int dy = k / 3 - 1, dx = k % 3 - 1;
            acc = __fadd_rn(acc, __fmul_rn(in(c, y + dy, x + dx), k == 4 ? b : a));
        }
        return ta_clamp01(__fmaf_rn(__fsub_rn(acc, v), f_alpha, v));  // add_(alpha=): fused
    }
    __device__ float op_value(int c, int y, int x) const {
        switch (op) {
            case kTaIdentity: return in(c, y, x);
            case kTaBrightness: return ta_clamp01(__fmul_rn(in(c, y, x), f_mul));
            case kTaColor:
                if (C == 1) return in(c, y, x);
                return ta_clamp01(__fmaf_rn(gray(y, x), f_alpha, __fmul_rn(in(c, y, x), f_mul)));
            case kTaContrast: return ta_clamp01(__fmaf_rn(s->mean, f_alpha, __fmul_rn(in(c, y, x), f_mul)));
            case kTaSharpness: return sharpen(c, y, x);
            case kTaPosterize: {
                const float levels = (float)(1 << (int)mag);
                const float q = floorf(__fmul_rn(in(c, y, x), levels));
                return __fmul_rn(q < 0.0f ? 0.0f : (q > levels - 1.0f ? levels - 1.0f : q), 1.0f / levels);
            }
            case kTaSolarize: {
                const float v = in(c, y, x);
                return v >= mag ? __fsub_rn(1.0f, v) : v;
            }
            case kTaAutoContrast: return ta_clamp01(__fdiv_rn(__fsub_rn(in(c, y, x), s->cmin[c]), s->cinv[c]));
            case kTaEqualize: return s->lut[c][ta_quantize(in(c, y, x))];
            case kTaInvert: return __fsub_rn(1.0f, in(c, y, x));
            default: return geometric(c, y, x);
        }
    }
    // kNorm: normalised into kBf16 | fp32 bits (the chain's last slot), else the fp32 bits of the op's value
    template <bool kBf16, bool kNorm>
    __device__ __forceinline__ uint32_t value(long long e) const {
        int c, p;
        if (nhwc) {
            p = (int)(e / C), c = (int)(e - (long long)p * C);
        } else {
            c = (int)(e / P), p = (int)(e - (long long)c * P);
        }
        if (nan) return kBf16 ? 0x7fc0u : 0x7fc00000u;
        const int y = p / w;
        float v = op_value(c, y, p - y * w);
        if (kNorm) v = __fdiv_rn(__fsub_rn(v, mean[c]), std[c]);
        return kBf16 ? (uint32_t)f32_to_bf16(v) : __float_as_uint(v);
    }
};

template <bool kWork, bool kBf16, bool kNorm>
struct TaCursor {
    const TaSample<kWork> &s;
    long long e;
    __device__ __forceinline__ uint32_t next() { return s.template value<kBf16, kNorm>(e++); }
};

// The cluster's statistics of the sample's op (Contrast, AutoContrast, Equalize) into s; every CTA calls it.
template <bool kWork>
__device__ void ta_statistics(const TaSample<kWork> &t, TaShared &s, cg::cluster_group &cluster) {
    const int rank = (int)cluster.block_rank(), n = (int)cluster.num_blocks();
    const int p0 = (int)((long long)t.P * rank / n), p1 = (int)((long long)t.P * (rank + 1) / n);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (t.op == kTaEqualize) {
        for (int k = threadIdx.x; k < 3 * 256; k += blockDim.x) (&s.hist[0][0])[k] = 0;
        __syncthreads();
        for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x)
            for (int c = 0; c < t.C; ++c) atomicAdd(&s.hist[c][ta_quantize(t.in(c, p / t.w, p % t.w))], 1u);
    } else if (t.op == kTaContrast) {
        __int128 acc = 0;
        for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
            float g = t.gray(p / t.w, p % t.w);
            g = g != g ? 0.0f : fminf(fmaxf(g, -2147483648.0f), 2147483648.0f);
            acc += f32_trunc_i128(__fmul_rn(g, 18446744073709551616.0f));
        }
        for (int o = 16; o; o >>= 1) {
            const unsigned long long lo = __shfl_down_sync(0xffffffffu, (unsigned long long)acc, o);
            const unsigned long long hi = __shfl_down_sync(0xffffffffu, (unsigned long long)((unsigned __int128)acc >> 64), o);
            acc += (__int128)(((unsigned __int128)hi << 64) | lo);
        }
        if (lane == 0) s.wsum[warp] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            __int128 sum = 0;
            for (int k = 0; k < kTaWarps; ++k) sum += s.wsum[k];
            s.sum = sum;
        }
    } else {  // AutoContrast: NaN values are not counted (fminf / fmaxf)
        float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x)
            for (int c = 0; c < t.C; ++c) {
                const float v = t.in(c, p / t.w, p % t.w);
                mn[c] = fminf(mn[c], v), mx[c] = fmaxf(mx[c], v);
            }
        for (int c = 0; c < 3; ++c) {
            for (int o = 16; o; o >>= 1) {
                mn[c] = fminf(mn[c], __shfl_down_sync(0xffffffffu, mn[c], o));
                mx[c] = fmaxf(mx[c], __shfl_down_sync(0xffffffffu, mx[c], o));
            }
            if (lane == 0) s.wmin[warp][c] = mn[c], s.wmax[warp][c] = mx[c];
        }
        __syncthreads();
        if (threadIdx.x < 3) {
            float a = INFINITY, b = -INFINITY;
            for (int k = 0; k < kTaWarps; ++k) a = fminf(a, s.wmin[k][threadIdx.x]), b = fmaxf(b, s.wmax[k][threadIdx.x]);
            s.mn[threadIdx.x] = a, s.mx[threadIdx.x] = b;
        }
    }
    cluster.sync();  // every CTA's partials are complete
    if (t.op == kTaEqualize) {
        for (int k = threadIdx.x; k < t.C * 256; k += blockDim.x) {
            unsigned int v = 0;
            for (int r = 0; r < n; ++r) v += (&cluster.map_shared_rank(&s, r)->hist[0][0])[k];
            (&s.total[0][0])[k] = v;
        }
    } else if (t.op == kTaContrast) {
        if (threadIdx.x == 0) {
            __int128 sum = 0;
            for (int r = 0; r < n; ++r) sum += cluster.map_shared_rank(&s, r)->sum;
            s.mean = (float)(i128_to_f64(sum) * 0x1p-64 / (double)t.P);
        }
    } else if (threadIdx.x < t.C) {
        const int c = threadIdx.x;
        float a = INFINITY, b = -INFINITY;
        for (int r = 0; r < n; ++r) {
            const TaShared *q = cluster.map_shared_rank(&s, r);
            a = fminf(a, q->mn[c]), b = fmaxf(b, q->mx[c]);
        }
        s.cmin[c] = a == b ? 0.0f : a;
        s.cinv[c] = a == b ? 1.0f : __fsub_rn(b, a);
    }
    cluster.sync();  // no CTA leaves while another reads its shared memory
    if (t.op == kTaEqualize && threadIdx.x < t.C) {  // torchvision's lut, one channel per thread
        const int c = threadIdx.x;
        unsigned int cum = 0, last = 0;
        for (int k = 0; k < 256; ++k)
            if (s.total[c][k]) last = k;
        const unsigned int step = ((unsigned int)t.P - s.total[c][last]) / 255u;
        for (int k = 0; k < 256; ++k) {
            unsigned int level = (unsigned int)k;
            if (step) {
                level = k == 0 ? 0u : min((cum + step / 2) / step, 255u);
                cum += s.total[c][k];
            }
            s.lut[c][k] = __fmul_rn((float)level, (float)(1.0 / 255.0));
        }
    }
    __syncthreads();
}

// Whether op row `row` makes its sample NaN: an op code outside [0, n_codes), or a Posterize magnitude outside (-1, 9).
__device__ __forceinline__ bool ta_bad_row(const int *row, int n_codes) {
    const int op = __ldg(row);
    const float mag = __int_as_float(__ldg(row + 1));
    return op < 0 || op >= n_codes || (op == kTaPosterize && !(mag > -1.0f && mag < 9.0f));
}

// One slot of a sample: the op of `row` on the sample's current buffer `cur`; the sample's elements [e0, e1) are
// written to dst from its element `first` on (kNorm: normalised into out's dtype, else fp32).  Every CTA of the
// cluster calls it.
template <bool kWork, bool kBf16, bool kNorm>
__device__ __forceinline__ void ta_slot(const TaArgs &a, TaShared &s, cg::cluster_group &cluster, const int *row,
                                        const float *cur, bool nan, void *dst, long long first, long long e0,
                                        long long e1) {
    TaSample<kWork> t;
    t.src = cur;
    t.s = &s;
    t.mean = a.mean, t.std = a.std;
    t.C = a.C, t.h = a.h, t.w = a.w, t.P = a.h * a.w, t.nhwc = a.nhwc, t.bilinear = a.bilinear;
    t.op = __ldg(row);
    t.mag = __int_as_float(__ldg(row + 1));
    for (int k = 0; k < 6; ++k) t.r[k] = __fdiv_rn(__int_as_float(__ldg(row + 2 + k)), 0.5f * (float)(k < 3 ? a.w : a.h));
    const double factor = 1.0 + (double)t.mag;
    t.f_mul = (float)factor, t.f_alpha = (float)(1.0 - factor);
    t.rot = 0;
    if (t.op == kTaRotate) {  // torchvision rotate's exact paths, on python's angle % 360
        double deg = fmod((double)t.mag, 360.0);
        if (deg < 0.0) deg += 360.0;
        t.rot = deg == 0.0 ? 4 : deg == 180.0 ? 2 : a.h != a.w ? 0 : deg == 90.0 ? 1 : deg == 270.0 ? 3 : 0;
    }
    t.nan = nan;
    if (!t.nan && (t.op == kTaContrast || t.op == kTaAutoContrast || t.op == kTaEqualize)) ta_statistics(t, s, cluster);
    image_store_run<kBf16>(dst, first, (int)(e1 - e0), [&](int k) { return TaCursor<kWork, kBf16, kNorm>{t, e0 + k}; });
}

// kChain: n_ops may exceed 1 (dmlb_image_auto_augment); the one-op kernel (dmlb_image_trivial_augment, and n_ops == 1)
// keeps only the last slot, which reads src through the non-coherent path.  The chain holds the state of every slot
// kind at once: two CTAs per SM give ptxas the registers to keep it without spilling.
template <bool kBf16, bool kChain>
__global__ void __launch_bounds__(kTaThreads, kChain ? 2 : 0) image_augment_kernel(const TaArgs a) {
    __shared__ TaShared s;
    cg::cluster_group cluster = cg::this_cluster();
    const int n = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const long long i = blockIdx.x / n;
    const int n_ops = kChain ? a.n_ops : 1;
    const int *rows = a.ops + 8LL * n_ops * i;
    const float *src = a.src + i * a.S;
    bool nan = __ldg(src) != __ldg(src);
    for (int k = 0; k < n_ops; ++k) nan = nan || ta_bad_row(rows + 8 * k, a.n_codes);
    const long long e0 = a.S * rank / n, e1 = a.S * (rank + 1) / n;
    int cur = -1;  // the sample's current buffer: src (-1) or work batch 0 / 1
    for (int k = 0; k + 1 < n_ops && !nan; ++k) {
        if (__ldg(rows + 8 * k) == kTaIdentity) continue;
        const int next = cur == 0 ? 1 : 0;
        float *dst = a.work + (next * a.batch + i) * a.S;
        if (cur < 0)
            ta_slot<false, false, false>(a, s, cluster, rows + 8 * k, src, false, dst, e0, e0, e1);
        else
            ta_slot<true, false, false>(a, s, cluster, rows + 8 * k, a.work + (cur * a.batch + i) * a.S, false, dst, e0,
                                        e0, e1);
        cluster.sync();  // every CTA's part of dst is written and visible to the cluster (release / acquire)
        cur = next;
    }
    const int *last = rows + 8 * (n_ops - 1);
    if (!kChain || cur < 0)
        ta_slot<false, kBf16, true>(a, s, cluster, last, src, nan, a.out, i * a.S + e0, e0, e1);
    else
        ta_slot<true, kBf16, true>(a, s, cluster, last, a.work + (cur * a.batch + i) * a.S, nan, a.out, i * a.S + e0, e0,
                                   e1);
}

static int ta_cluster(long long pixels) {
    const long long n = (pixels + kTaPixelsPerCta - 1) / kTaPixelsPerCta;
    return (int)(n < kTaMaxCluster ? n : kTaMaxCluster);
}

template <bool kBf16, bool kChain>
static int launch_augment(int cluster, cudaStream_t st, const TaArgs &a) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(a.batch * cluster));
    cfg.blockDim = dim3(kTaThreads);
    cfg.stream = st;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)cluster, attr.val.clusterDim.y = 1, attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, image_augment_kernel<kBf16, kChain>, a);
    const int r = launched();
    return e != cudaSuccess ? -(int)e : r;
}

static bool overlaps(const void *p, long long p_bytes, const void *q, long long q_bytes) {
    const uintptr_t p0 = (uintptr_t)p, q0 = (uintptr_t)q;
    return p_bytes > 0 && q_bytes > 0 && p0 < q0 + (uintptr_t)q_bytes && q0 < p0 + (uintptr_t)p_bytes;
}

// The checks and the launch of both op-chain entries (n_codes: 14 for TrivialAugment's ops, 15 with Invert).
static int augment(const float *src, float *work, const int32_t *ops, int n_ops, int n_codes, int64_t batch, int32_t C,
                   int32_t h, int32_t w, int bilinear, const dmlb_image_norm *norm, void *out, int out_bf16,
                   int channels_last, void *stream) {
    if (batch < 0 || batch > kTaMaxBatch || !norm || (C != 1 && C != 3) || h < 1 || w < 1 || h > kTaMaxSide ||
        w > kTaMaxSide || (long long)h * w > kTaMaxPixels || (bilinear != 0 && bilinear != 1) || n_ops < 1 ||
        n_ops > kTaMaxChain)
        return DMLB_EINVAL;
    TaArgs a;
    if (!pack_norm(norm, C, a.mean, a.std)) return DMLB_EINVAL;
    if (batch > 0 && (!src || !ops || !out || (n_ops > 1 && !work))) return DMLB_EINVAL;
    const long long S = (long long)C * h * w;
    const long long src_bytes = batch * S * 4, out_bytes = batch * S * (out_bf16 ? 2 : 4);
    const long long work_bytes = n_ops > 1 ? (n_ops > 2 ? 2 : 1) * src_bytes : 0;
    if (overlaps(src, src_bytes, out, out_bytes) || overlaps(work, work_bytes, src, src_bytes) ||
        overlaps(work, work_bytes, ops, batch * n_ops * 32) || overlaps(work, work_bytes, out, out_bytes))
        return DMLB_EINVAL;
    if (((uintptr_t)src & 3) != 0 || ((uintptr_t)ops & 3) != 0 || ((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0 ||
        (n_ops > 1 && ((uintptr_t)work & 3) != 0))
        return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    a.src = src;
    a.work = n_ops > 1 ? work : nullptr;
    a.ops = ops;
    a.out = out;
    a.S = S, a.batch = batch;
    a.n_ops = n_ops, a.n_codes = n_codes;
    a.C = C, a.h = h, a.w = w, a.nhwc = channels_last ? 1 : 0, a.bilinear = bilinear;
    const int cluster = ta_cluster((long long)h * w);
    cudaStream_t st = (cudaStream_t)stream;
    if (n_ops > 1) return out_bf16 ? launch_augment<true, true>(cluster, st, a) : launch_augment<false, true>(cluster, st, a);
    return out_bf16 ? launch_augment<true, false>(cluster, st, a) : launch_augment<false, false>(cluster, st, a);
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

int dmlb_image_batch_u8(const uint8_t *images, const int64_t *idx, const int32_t *windows, int64_t batch, int32_t H,
                        int32_t W, int32_t C, int32_t out_h, int32_t out_w, int32_t pad, const dmlb_image_norm *norm,
                        void *out, int out_bf16, int channels_last, void *stream) {
    if (batch < 0 || !norm || C < 1 || C > 4 || H < 1 || W < 1 || out_h < 1 || out_w < 1 || pad < 0) return DMLB_EINVAL;
    const long long dy = (long long)H + 2LL * pad - out_h, dx = (long long)W + 2LL * pad - out_w;
    if (dy < 0 || dx < 0) return DMLB_EINVAL;
    ImageArgs a;
    if (!pack_norm(norm, C, a.mean, a.std)) return DMLB_EINVAL;
    if (batch > 0 && (!images || !idx || !windows || !out)) return DMLB_EINVAL;
    const long long rowcap = ((long long)out_w * C + 15) / 16 * 16 + 16;
    if (rowcap > kImageMaxRowBytes) return DMLB_EINVAL;
    if (((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0 || ((uintptr_t)windows & 3) != 0) return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    a.images = images;
    a.idx = (const long long *)idx;
    a.windows = windows;
    a.out = out;
    a.batch = batch;
    a.sample_bytes = (long long)H * W * C;
    a.H = H, a.W = W, a.C = C, a.oh = out_h, a.ow = out_w, a.pad = pad;
    a.dy = dy, a.dx = dx;
    const int max_rows = (int)(kImageBandBytes / rowcap) > 0 ? (int)(kImageBandBytes / rowcap) : 1;
    a.bands = (out_h + max_rows - 1) / max_rows;
    a.rows = (out_h + a.bands - 1) / a.bands;
    a.rowcap = (int)rowcap;
    const int grid = band_grid(batch * a.bands, kImageCtasPerSm);
    const size_t smem = (size_t)a.rows * a.rowcap;
    const bool vec_load = ((uintptr_t)images & 15) == 0;
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_layout(out_bf16, channels_last, [&](auto bf16, auto nhwc) {
        return launch_image<decltype(bf16)::value, decltype(nhwc)::value>(vec_load, grid, smem, st, a);
    });
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
    ResampleArgs a;
    if (!pack_norm(norm, C, a.mean, a.std)) return DMLB_EINVAL;
    if (batch > 0 && (!images || !idx || !boxes || !out)) return DMLB_EINVAL;
    if (((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0 || ((uintptr_t)boxes & 3) != 0) return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    const ResamplePlan p = resample_plan(H, W, C, resize_h, resize_w, out_h, out_w, H);
    a.images = images;
    a.idx = (const long long *)idx;
    a.geom = boxes;
    a.extents = nullptr;
    a.sample_bytes = (long long)H * W * C;
    a.H = H, a.W = W, a.rh = resize_h, a.rw = resize_w, a.win_top = win_top, a.win_left = win_left;
    return resample_launch<LaunchGeometry>(a, p, batch, C, out_h, out_w, out, out_bf16, channels_last, stream);
}

int dmlb_image_resample_ragged_u8(const uint8_t *store, int64_t store_bytes, const dmlb_image_extent *extents,
                                  const int64_t *idx, const int32_t *geom, int64_t batch, int32_t C, int32_t bound_h,
                                  int32_t bound_rh, int32_t bound_w, int32_t bound_rw, int32_t out_h, int32_t out_w,
                                  const dmlb_image_norm *norm, void *out, int out_bf16, int channels_last,
                                  void *stream) {
    if (batch < 0 || store_bytes < 0 || !norm || C < 1 || C > 4) return DMLB_EINVAL;
    for (int32_t side : {bound_h, bound_rh, bound_w, bound_rw, out_h, out_w})
        if (side < 1 || side > kResampleMaxSide) return DMLB_EINVAL;
    if ((long long)bound_h > (long long)kResampleMaxScale * bound_rh ||
        (long long)bound_w > (long long)kResampleMaxScale * bound_rw)
        return DMLB_EINVAL;
    if ((long long)out_w * C > kResampleMaxRowElems) return DMLB_EINVAL;
    ResampleArgs a;
    if (!pack_norm(norm, C, a.mean, a.std)) return DMLB_EINVAL;
    if (batch > 0 && (!store || !extents || !idx || !geom || !out)) return DMLB_EINVAL;
    if (((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0 || ((uintptr_t)geom & 3) != 0 || ((uintptr_t)extents & 7) != 0)
        return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    const ResamplePlan p = resample_plan(bound_h, bound_w, C, bound_rh, bound_rw, out_h, out_w, kResampleMaxSide);
    a.images = store;
    a.idx = (const long long *)idx;
    a.geom = geom;
    a.extents = extents;
    a.sample_bytes = store_bytes;
    a.H = a.W = a.rh = a.rw = a.win_top = a.win_left = 0;
    return resample_launch<TableGeometry>(a, p, batch, C, out_h, out_w, out, out_bf16, channels_last, stream);
}

int dmlb_image_mix(const float *src, const int64_t *idx, const int64_t *labels, const int32_t *erase, const float *fill,
                   int64_t batch, int32_t C, int32_t h, int32_t w, int mode, double lam, int32_t y1, int32_t y2,
                   int32_t x1, int32_t x2, int32_t num_classes, void *out, int out_bf16, int channels_last,
                   void *targets, void *stream) {
    if (batch < 0 || C < 1 || C > 4 || h < 1 || w < 1 || h > kMixMaxSide || w > kMixMaxSide) return DMLB_EINVAL;
    if (mode < 0 || mode > 2 || !(lam >= 0.0 && lam <= 1.0)) return DMLB_EINVAL;
    if (y1 < 0 || y1 > y2 || y2 > h || x1 < 0 || x1 > x2 || x2 > w) return DMLB_EINVAL;
    if (mode != 0 && num_classes < 1) return DMLB_EINVAL;
    if (batch > 0 && (!src || !idx || !labels || !out || !targets || (erase && !fill))) return DMLB_EINVAL;
    const long long S = (long long)C * h * w;
    if (((uintptr_t)out & (out_bf16 ? 1 : 3)) != 0 || ((uintptr_t)src & 3) != 0 || ((uintptr_t)erase & 3) != 0 ||
        ((uintptr_t)targets & (mode == 0 ? 7 : 3)) != 0)
        return DMLB_EALIGN;
    if (batch == 0) return DMLB_OK;

    MixArgs a;
    a.src = src;
    a.idx = (const long long *)idx;
    a.labels = (const long long *)labels;
    a.erase = erase;
    a.out = out;
    a.targets = targets;
    a.batch = batch;
    a.S = S;
    a.h = h, a.w = w, a.C = C, a.nhwc = channels_last ? 1 : 0, a.mode = mode;
    a.y1 = mode == 2 ? y1 : 0, a.y2 = mode == 2 ? y2 : 0, a.x1 = mode == 2 ? x1 : 0, a.x2 = mode == 2 ? x2 : 0;
    a.K = mode == 0 ? 1 : num_classes;
    a.w_prev = (float)(1.0 - lam);
    a.w_cur = (float)lam;
    for (int c = 0; c < 4; ++c) a.fill[c] = erase && c < C ? fill[c] : 0.0f;
    const int V = out_bf16 ? 8 : 4;
    const bool vec = S % V == 0 && ((uintptr_t)src & 15) == 0 && ((uintptr_t)out & 15) == 0;
    a.nvec = vec ? S / V : S;
    // segments: enough of them to give every SM kMixCtasPerSm CTAs, none shorter than one unrolled group
    const long long gx = (a.nvec + kMixThreads - 1) / kMixThreads;
    long long nseg = ((long long)sm_count() * kMixCtasPerSm + gx - 1) / gx;
    const long long max_seg = (batch + kMixUnroll - 1) / kMixUnroll;
    nseg = nseg < max_seg ? nseg : max_seg;  // at most sm_count * kMixCtasPerSm, far below the grid's y limit
    a.seglen = (int)((batch + nseg - 1) / nseg);
    nseg = (batch + a.seglen - 1) / a.seglen;
    const dim3 grid((unsigned)gx, (unsigned)nseg);  // gx <= 2^32 / 256 at the largest accepted sample
    cudaStream_t st = (cudaStream_t)stream;
    if (out_bf16) return vec ? launch_mix<true, 8>(grid, st, a) : launch_mix<true, 1>(grid, st, a);
    return vec ? launch_mix<false, 4>(grid, st, a) : launch_mix<false, 1>(grid, st, a);
}

int dmlb_image_trivial_augment(const float *src, const int32_t *ops, int64_t batch, int32_t C, int32_t h, int32_t w,
                               int bilinear, const dmlb_image_norm *norm, void *out, int out_bf16, int channels_last,
                               void *stream) {
    return augment(src, nullptr, ops, 1, kTaOps, batch, C, h, w, bilinear, norm, out, out_bf16, channels_last, stream);
}

int dmlb_image_auto_augment(const float *src, float *work, const int32_t *ops, int32_t n_ops, int64_t batch, int32_t C,
                            int32_t h, int32_t w, int bilinear, const dmlb_image_norm *norm, void *out, int out_bf16,
                            int channels_last, void *stream) {
    return augment(src, work, ops, n_ops, kTaOps + 1, batch, C, h, w, bilinear, norm, out, out_bf16, channels_last,
                   stream);
}

}  // extern "C"
