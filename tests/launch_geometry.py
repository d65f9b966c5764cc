"""Host-side launch decisions of libdmlb, restated in Python as functions of the device's SM count.

Every kernel picks its grid (and sometimes its loop shape or protocol) from the message size and the SM count, so the
sizes where a kernel changes regime move with the SM count and with any retune.  The GPU tests take their boundary sizes
from here, computed for the device they run on, and check with a profiler trace (helpers.dmlb_launches) that each size
reached the kernel and grid named here.  The constants below are copied verbatim from the sources listed in PINS;
tests/test_launch_geometry.py checks that each copied line still appears there, so a retune fails the CPU tier instead of
silently moving the GPU test sizes off their boundaries.
"""

# (source file relative to dmlcloud_b200/csrc, declaration line copied verbatim)
PINS = [
    ('dmlb_common.cuh', 'constexpr int kThreads = 512;'),
    ('dmlb_common.cuh', 'if (want <= cap) return (int)want;'),
    ('dmlb_common.cuh', 'size_t sweeps = (want + cap - 1) / cap;'),
    ('dmlb_common.cuh', 'return (int)((want + sweeps - 1) / sweeps);'),
    ('bucket_kernels.cu', 'constexpr size_t kTmaMinElems = 32u << 20;'),
    ('bucket_kernels.cu', 'constexpr int kUnroll = 4;      // independent vector loads a thread issues before its first store'),
    ('bucket_kernels.cu', 'constexpr int kCtasPerSm = 4;'),
    ('bucket_kernels.cu', 'if (want <= 2 * cap) {  // at most two waves: balance the SMs (see stream_kernel)'),
    ('bucket_kernels.cu', 'size_t g = want < sms ? (want < 1 ? 1 : want) : ((want + sms - 1) / sms) * sms;'),
    ('bucket_kernels.cu', 'if (g > cap) g = cap;'),
    ('bucket_kernels.cu', 'chunk = (nvec + g - 1) / g;'),
    ('bucket_kernels.cu', 'grid = stream_grid(nvec, kUnroll, kCtasPerSm);'),
    ('optim_kernels.cu', 'const int grid = stream_grid(n / 4, 2, 2);'),
    ('optim_kernels.cu', 'const int grid = stream_grid(n, 1, 2);'),
    ('peer_comm.cuh', 'constexpr int kMaxCtas = 264;  // 2 per SM on 132 SMs (launches use at most 2 x the device\'s SM count)'),
    ('peer_comm.cuh', 'constexpr int kCommThreads = 256;'),
    ('peer_comm.cuh', 'constexpr size_t kMetricStageBytes = 16384;  // per half: 16-byte header + 16 B per exchanged cell'),
    ('peer_comm.cuh', 'constexpr int kStepMetricMaxCells = (int)(kMetricStageBytes / 16) - 1;'),
    ('peer_comm.cuh', 'constexpr size_t kLLMaxPayload = 256 * 1024;'),
    ('peer_comm.cu', 'constexpr size_t kOneshotMaxBytes = 512 * 1024;'),
    ('peer_comm.cu', 'const bool oneshot = !nvls && (W == 1 || algo == 1 || algo == 5 || (algo == 0 && (bytes <= kOneshotMaxBytes || W <= 2)));'),
    ('peer_comm.cu', 'const int EL = wire == DMLB_WIRE_BF16 ? 4 : 2;'),
    ('peer_comm.cu', 'if (oneshot && W > 1 && algo != 5 && bytes <= kLLMaxPayload) {'),
    ('peer_comm.cu', 'size_t want = (n_lines + kCommThreads - 1) / kCommThreads;  // one line per thread while the grid can grow'),
    ('peer_comm.cu', 'const int kU = W <= 2 ? 4 : (W <= 4 ? 2 : 1);'),
    ('peer_comm.cu', 'const size_t items = oneshot ? nvec : (nvec + W - 1) / W;  // vectors a CTA grid is spread over'),
    ('peer_comm.cu', 'size_t want = (items + (size_t)kCommThreads * kU - 1) / ((size_t)kCommThreads * kU);'),
    ('peer_comm.cu', 'const int grid = n_data + (metrics ? 1 : 0);'),
    ('peer_comm.cu', 'size_t cap = (size_t)min(kMaxCtas, sm_count() * 2) - 1;'),
    ('metric_kernels.cu', 'constexpr int kExchangeGrid = 8;  // CTAs of an exchanging reduce: a CONSTANT, so ranks with different selections still pair'),
    ('metric_kernels.cu', 'int grid = (end - begin + 255) / 256;'),
    ('metric_kernels.cu', 'if (grid > sm_count()) grid = sm_count();'),
    ('metric_kernels.cu', 'metric_reset_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>'),
    ('shard_kernels.cu', 'long long cap = (long long)sm_count() * 8;'),
    ('shard_kernels.cu', 'int grid = grid_for(batch * vpr, 256);'),
]

K_THREADS = 512
K_TMA_MIN_ELEMS = 32 << 20
K_UNROLL = 4
K_CTAS_PER_SM = 4
K_MAX_CTAS = 264
K_COMM_THREADS = 256
K_METRIC_STAGE_BYTES = 16384
STEP_METRIC_MAX_CELLS = K_METRIC_STAGE_BYTES // 16 - 1
K_LL_MAX_PAYLOAD = 256 * 1024
K_ONESHOT_MAX_BYTES = 512 * 1024
K_EXCHANGE_GRID = 8
RESET_THREADS = 256
SHARD_THREADS = 256
SHARD_CTAS_PER_SM = 8


def cdiv(a, b):
    return -(-a // b)


def stream_grid(nvec, per_thread, ctas_per_sm, sms):
    """dmlb_common.cuh stream_grid: a grid-stride grid whose sweeps are (almost) all full."""
    want = max(1, cdiv(nvec, K_THREADS * per_thread))
    cap = sms * ctas_per_sm
    if want <= cap:
        return want
    sweeps = cdiv(want, cap)
    return cdiv(want, sweeps)


# ---- bucket_kernels.cu launch_stream (fp32-side functors: 4 elements per vector item) --------------------------------
def launch_stream(n, head, sms):
    """(grid, chunk) of stream_kernel for n elements whose first `head` (0..3) are the scalar head; chunk 0 = grid-stride
    sweeps, chunk > 0 = every CTA owns `chunk` consecutive vectors."""
    h = min(head, n)
    nvec = (n - h) // 4
    per_cta = K_THREADS * K_UNROLL
    want = cdiv(nvec, per_cta)
    cap = sms * K_CTAS_PER_SM
    if want <= 2 * cap:
        g = max(1, want) if want < sms else cdiv(want, sms) * sms
        g = min(g, cap)
        return g, max(1, cdiv(nvec, g))
    return stream_grid(nvec, K_UNROLL, K_CTAS_PER_SM, sms), 0


def stream_sizes(sms):
    """Aligned (head 0) element counts at the edges of launch_stream's regimes."""
    per_cta = K_THREADS * K_UNROLL
    cap = sms * K_CTAS_PER_SM
    return {
        'last_first_wave': 4 * sms * per_cta + 3,       # want == sms: one CTA per SM, the grid is not rounded
        'first_rounded_grid': 4 * (sms * per_cta + 1),  # want == sms + 1: grid rounded up to a multiple of sms
        'last_chunked': 4 * 2 * cap * per_cta + 3,      # want == 2 * cap: the last two-wave chunked launch
        'first_grid_stride': 4 * (2 * cap * per_cta + 1),  # more than two waves: grid-stride sweeps
    }


# ---- optim_kernels.cu Adam / SGD ---------------------------------------------------------------------------------------
def optim_grid(n, vector, sms):
    return stream_grid(n // 4, 2, 2, sms) if vector else stream_grid(n, 1, 2, sms)


def optim_sweeps(n, vector, sms):
    items, per_thread = (n // 4, 2) if vector else (n, 1)
    return cdiv(items, optim_grid(n, vector, sms) * K_THREADS * per_thread)


def optim_sizes(sms):
    return {'first_multi_sweep': 4 * (2 * sms * K_THREADS * 2 + 1)}  # vector path: more vectors than one sweep covers


# ---- peer_comm.cu dmlb_comm_allreduce ----------------------------------------------------------------------------------
def allreduce_plan(n, wire_bf16, world, sms, algo=0, metrics=False):
    """(protocol, grid, n_data) of dmlb_comm_allreduce without multicast: protocol is 'll', 'oneshot' or 'twoshot'."""
    E = 8 if wire_bf16 else 4
    nvec = cdiv(n, E)
    nbytes = nvec * 16
    cap = min(K_MAX_CTAS, 2 * sms) - 1
    oneshot = world == 1 or algo in (1, 5) or (algo == 0 and (nbytes <= K_ONESHOT_MAX_BYTES or world <= 2))
    if oneshot and world > 1 and algo != 5 and nbytes <= K_LL_MAX_PAYLOAD:
        EL = 4 if wire_bf16 else 2
        want = min(cdiv(cdiv(n, EL), K_COMM_THREADS), cap)
        n_data = 0 if n == 0 else max(1, want)
        return 'll', n_data + int(metrics), n_data
    kU = allreduce_ku(world)
    items = nvec if oneshot else cdiv(nvec, world)
    want = min(cdiv(items, K_COMM_THREADS * kU), cap)
    n_data = 0 if n == 0 else max(1, want)
    return ('oneshot' if oneshot else 'twoshot'), n_data + int(metrics), n_data


def allreduce_ku(world):
    return 4 if world <= 2 else (2 if world <= 4 else 1)


def allreduce_sizes(wire_bf16, world, sms):
    """Element counts on both sides of each protocol switch and at the first capped grid."""
    E = 8 if wire_bf16 else 4
    cap = min(K_MAX_CTAS, 2 * sms) - 1
    kU = allreduce_ku(world)
    out = {
        'll_max': K_LL_MAX_PAYLOAD // 16 * E,
        'll_max_plus_1': K_LL_MAX_PAYLOAD // 16 * E + 1,
        # one-shot forced (algo 1) or automatic (W <= 2): the data grid reaches its cap
        'first_capped_oneshot': cap * K_COMM_THREADS * kU * E + 1,
    }
    if world > 2:
        out['oneshot_max'] = K_ONESHOT_MAX_BYTES // 16 * E
        out['twoshot_min'] = K_ONESHOT_MAX_BYTES // 16 * E + 1
        out['first_capped_twoshot'] = world * cap * K_COMM_THREADS * kU * E + 1
    return out


# ---- metric_kernels.cu --------------------------------------------------------------------------------------------------
def metric_reset_grid(cells, sms):
    return min(cdiv(cells, RESET_THREADS), sms)


def metric_sizes(sms):
    return {
        'reset_first_capped': RESET_THREADS * sms + 1,                     # one reset of more cells than its grid covers
        'exchange_first_looping': K_EXCHANGE_GRID * K_COMM_THREADS + 1,    # a CTA of the exchanging reduce loops
    }


# ---- shard_kernels.cu ---------------------------------------------------------------------------------------------------
def shard_grid(work, sms):
    return max(1, min(cdiv(work, SHARD_THREADS), SHARD_CTAS_PER_SM * sms))
