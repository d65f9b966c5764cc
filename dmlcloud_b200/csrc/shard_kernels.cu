// Device-resident data-shard iterator kernels (SURVEY §8f-1).
//
// Reference: util/data.py:11-30 shard_indices (`indices[rank::world]` after the optional MT19937 shuffle and tail drop)
// and examples/mnist.py:16-21 (torchvision ToTensor + Normalize((0.1307,), (0.3081,)) + DataLoader batching, on the host).
// Here the whole uint8 dataset stays in HBM (MNIST: 47 MB of 180 GB); the epoch permutation is uploaded once per epoch
// (bit-exact host computation — the same numpy MT19937 stream the reference uses) and each step is one gather kernel:
//   out[i, :] = (float(images[idx[i], :]) / 255 - mean) / std                      784 B read, 3136 (fp32) B written / sample
// HBM-bound byte work: 16 pixels (one 128-bit load) per thread, 4x 128-bit stores, rows found through idx[] (L2-resident).
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
template <bool kVecLoad, bool kNHWC>
struct ImageCursor {
    const ImageBand<kVecLoad> &b;
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
                return ImageCursor<kVecLoad, true>{band, p / ow, p - (p / ow) * ow, k - p * C};
            });
        } else {
            for (int c = 0; c < a.C; ++c) {
                const int ow = a.ow;
                image_store_run<kBf16>(a.out, (i * a.C + c) * plane + (long long)y0 * ow, nr * ow, [&](int k) {
                    return ImageCursor<kVecLoad, false>{band, k / ow, k - (k / ow) * ow, c};
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

}  // extern "C"
