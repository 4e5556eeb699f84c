// extern "C" boundary of libjaero_b200.so (declared in include/jaero_b200.h).
// Host-side object management only: device allocation, staging copies, stream ordering, kernel
// launches. No CPU implementation of any DSP lives here — without a CUDA device every create
// call fails loudly.
#include "../../include/jaero_b200.h"
#include "common.cuh"
#include "viterbi.cuh"
#include "demod.cuh"
#include "demod_stages.cuh"                   // msk_half_symbol_delay
#include "prefilter.cuh"
#include "burst.cuh"
#include "frame_layers.cuh"
#include "ddc.cuh"
#include "scan.cuh"
#include "resample.cuh"
#include "ident.cuh"
#include <cstring>
#include <complex>
#include <climits>
#include <cstdlib>
#include <initializer_list>
#include <new>
#include <numeric>
#include <vector>

namespace jb {
static thread_local std::string g_err;
void set_error(const std::string &m) { g_err = m; }
int cuda_fail(cudaError_t e, const char *what, const char *file, int line)
{
    char buf[512];
    snprintf(buf, sizeof buf, "CUDA error %d (%s) at %s:%d in %s", (int)e, cudaGetErrorString(e), file, line, what);
    g_err = buf;
    return JAERO_E_CUDA;
}
} // namespace jb
using namespace jb;

// A create call that fails half-way (any JB_CUDA early return) hands the partly built object to its destroy function.
template <class T> struct CreateGuard {
    T *obj = nullptr; void (*destroy)(T *);
    explicit CreateGuard(void (*d)(T *)) : destroy(d) {}
    ~CreateGuard() { if (obj) destroy(obj); }
    // The first steps of every create: a valid device, a value-initialised (all-zero) object and its non-blocking stream.
    // `fn` prefixes the error text.
    int begin(const char *fn, int device)
    {
        int ndev = 0;
        JB_CUDA(cudaGetDeviceCount(&ndev));
        if (device < 0 || device >= ndev) { set_error(std::string(fn) + ": no such CUDA device"); return JAERO_E_CUDA; }
        JB_CUDA(cudaSetDevice(device));
        obj = new (std::nothrow) T();
        if (!obj) { set_error("out of host memory"); return JAERO_E_ARG; }
        obj->device = device;
        JB_CUDA(cudaStreamCreateWithFlags(&obj->stream, cudaStreamNonBlocking));
        return JAERO_OK;
    }
    T *release() { T *o = obj; obj = nullptr; return o; }
    CreateGuard(const CreateGuard &) = delete;
    CreateGuard &operator=(const CreateGuard &) = delete;
};

// *_sync: waits for the object's queued work
template <class O> int sync_stream(O *o)
{
    if (!o) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(o->device));
    JB_CUDA(cudaStreamSynchronize(o->stream));
    return JAERO_OK;
}
// *_set_stream: the work queued on the old stream drains first; a null stream goes back to the object's own
template <class O> int switch_stream(O *o, void *cuda_stream)
{
    int r = sync_stream(o); if (r) return r;
    o->stream = cuda_stream ? (cudaStream_t)cuda_stream : o->own_stream;
    return JAERO_OK;
}

struct jaero_viterbi {
    int n_channels, pad, device;
    cudaStream_t stream;
    uint8_t *d_overlap; int *d_overlap_len; int *d_renorm;
    uint8_t *d_soft, *d_bits; size_t soft_cap, bits_cap;
    int *d_valid;
    int64_t launches;
};

extern "C" {

const char *jaero_last_error(void) { return g_err.c_str(); }
int jaero_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// ------------------------------------------------------------------ Viterbi
int jaero_viterbi_create(int n_channels, int paddinglength, int device, jaero_viterbi **out)
{
    if (!out || n_channels <= 0 || paddinglength < 0 || (paddinglength & 1)) { set_error("jaero_viterbi_create: bad argument"); return JAERO_E_ARG; }
    CreateGuard<jaero_viterbi> guard(jaero_viterbi_destroy);
    int r = guard.begin("jaero_viterbi_create", device); if (r) return r;
    jaero_viterbi *v = guard.obj;
    v->n_channels = n_channels; v->pad = paddinglength;
    JB_CUDA(cudaMalloc(&v->d_overlap, (size_t)n_channels * 64));
    JB_CUDA(cudaMalloc(&v->d_overlap_len, (size_t)n_channels * sizeof(int)));
    JB_CUDA(cudaMalloc(&v->d_renorm, (size_t)n_channels * sizeof(int)));
    JB_CUDA(cudaMalloc(&v->d_valid, (size_t)n_channels * sizeof(int)));
    JB_CUDA(cudaMemsetAsync(v->d_overlap, 0, (size_t)n_channels * 64, v->stream));
    JB_CUDA(cudaMemsetAsync(v->d_overlap_len, 0, (size_t)n_channels * sizeof(int), v->stream));
    JB_CUDA(cudaMemsetAsync(v->d_renorm, 0, (size_t)n_channels * sizeof(int), v->stream));
    *out = guard.release();
    return JAERO_OK;
}
void jaero_viterbi_destroy(jaero_viterbi *v)
{
    if (!v) return;
    cudaSetDevice(v->device);
    cudaStreamSynchronize(v->stream);
    cudaFree(v->d_overlap); cudaFree(v->d_overlap_len); cudaFree(v->d_renorm); cudaFree(v->d_valid); cudaFree(v->d_soft); cudaFree(v->d_bits);
    cudaStreamDestroy(v->stream);
    delete v;
}
int jaero_viterbi_reset(jaero_viterbi *v)
{
    if (!v) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(v->device));
    JB_CUDA(cudaMemsetAsync(v->d_overlap_len, 0, (size_t)v->n_channels * sizeof(int), v->stream));
    return JAERO_OK;
}
int jaero_viterbi_sync(jaero_viterbi *v) { return sync_stream(v); }
int64_t jaero_viterbi_launch_count(const jaero_viterbi *v) { return v ? v->launches : 0; }

static int vit_check(jaero_viterbi *v, size_t n_soft, int cols)
{
    if (!v) { set_error("null handle"); return JAERO_E_ARG; }
    if (n_soft < 32 || (n_soft & 1) || n_soft > 60000) { set_error("viterbi: n_soft must be even, 32..60000"); return JAERO_E_ARG; }
    if (cols < 0 || (cols > 0 && (size_t)cols * 64 != n_soft)) { set_error("viterbi: interleaver_cols*64 must equal n_soft"); return JAERO_E_ARG; }
    return JAERO_OK;
}
int jaero_viterbi_decode_continuous_device(jaero_viterbi *v, const uint8_t *d_soft, size_t n_soft, int cols, uint8_t *d_bits, int32_t *d_n_valid)
{
    int r = vit_check(v, n_soft, cols); if (r) return r;
    JB_CUDA(cudaSetDevice(v->device));
    if (viterbi_launch(d_soft, (int)n_soft, cols, 0, v->pad, v->d_overlap, v->d_overlap_len, v->d_renorm, d_bits, d_n_valid, v->n_channels, v->stream)) return JAERO_E_CUDA;
    v->launches++;
    return JAERO_OK;
}
static int vit_stage(jaero_viterbi *v, size_t n_soft)
{
    size_t need = (size_t)v->n_channels * n_soft;
    if (need > v->soft_cap) { cudaFree(v->d_soft); v->d_soft = 0; JB_CUDA(cudaMalloc(&v->d_soft, need)); v->soft_cap = need; }
    size_t needb = (size_t)v->n_channels * (n_soft / 2);
    if (needb > v->bits_cap) { cudaFree(v->d_bits); v->d_bits = 0; JB_CUDA(cudaMalloc(&v->d_bits, needb)); v->bits_cap = needb; }
    return JAERO_OK;
}
int jaero_viterbi_decode_continuous(jaero_viterbi *v, const uint8_t *soft, size_t n_soft, int cols, uint8_t *bits_out, int32_t *n_valid)
{
    int r = vit_check(v, n_soft, cols); if (r) return r;
    if (!soft || !bits_out) { set_error("null buffer"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(v->device));
    r = vit_stage(v, n_soft); if (r) return r;
    JB_CUDA(cudaMemcpyAsync(v->d_soft, soft, (size_t)v->n_channels * n_soft, cudaMemcpyHostToDevice, v->stream));
    r = jaero_viterbi_decode_continuous_device(v, v->d_soft, n_soft, cols, v->d_bits, v->d_valid); if (r) return r;
    JB_CUDA(cudaMemcpyAsync(bits_out, v->d_bits, (size_t)v->n_channels * (n_soft / 2), cudaMemcpyDeviceToHost, v->stream));
    if (n_valid) JB_CUDA(cudaMemcpyAsync(n_valid, v->d_valid, (size_t)v->n_channels * sizeof(int), cudaMemcpyDeviceToHost, v->stream));
    JB_CUDA(cudaStreamSynchronize(v->stream));
    return JAERO_OK;
}
int jaero_viterbi_decode_block(jaero_viterbi *v, const uint8_t *soft, size_t n_soft, uint8_t *bits_out)
{
    int r = vit_check(v, n_soft, 0); if (r) return r;
    if (!soft || !bits_out) { set_error("null buffer"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(v->device));
    r = vit_stage(v, n_soft); if (r) return r;
    JB_CUDA(cudaMemcpyAsync(v->d_soft, soft, (size_t)v->n_channels * n_soft, cudaMemcpyHostToDevice, v->stream));
    if (viterbi_launch(v->d_soft, (int)n_soft, 0, 1, 0, v->d_overlap, v->d_overlap_len, v->d_renorm, v->d_bits, v->d_valid, v->n_channels, v->stream)) return JAERO_E_CUDA;
    v->launches++;
    JB_CUDA(cudaMemcpyAsync(bits_out, v->d_bits, (size_t)v->n_channels * (n_soft / 2), cudaMemcpyDeviceToHost, v->stream));
    JB_CUDA(cudaStreamSynchronize(v->stream));
    return JAERO_OK;
}

} // extern "C"

// ====================================================================== demodulator batches
#include <cmath>
#include <algorithm>

namespace {

// RootRaisedCosine::design (JAERO/DSP.h:316-338): closed-form RRC taps, firsize forced odd.
std::vector<double> rrc_taps(double alpha, int firsize, double samplerate, double symbol_freq)
{
    if ((firsize % 2) == 0) firsize += 1;
    std::vector<double> pts(firsize);
    const double T = (samplerate) / (symbol_freq);
    for (int i = 0; i < firsize; i++) {
        if (i == ((firsize - 1) / 2)) pts[i] = (4.0 * alpha + M_PI - M_PI * alpha) / (M_PI * sqrt(T));
        else {
            const double fi = (((double)i) - ((double)(firsize - 1)) / 2.0);
            if (fabs(1.0 - pow(4.0 * alpha * fi / T, 2)) < 0.0000000001)
                pts[i] = (alpha * ((M_PI - 2.0) * cos(M_PI / (4.0 * alpha)) + (M_PI + 2.0) * sin(M_PI / (4.0 * alpha))) / (M_PI * sqrt(2.0 * T)));
            else
                pts[i] = (4.0 * alpha / (M_PI * sqrt(T)) * (cos((1.0 + alpha) * M_PI * fi / T) + T / (4.0 * alpha * fi) * sin((1.0 - alpha) * M_PI * fi / T)) / (1.0 - pow(4.0 * alpha * fi / T, 2)));
        }
    }
    return pts;
}

// Delay<T>::update interpolation weight (JAERO/DSP.h:357-374) for every ring position, w[0 .. ceil(fractdelay)]. The kernels
// keep the delay line as a shift register; the weight the reference derives from (buffptr - fractdelay) can differ in the last
// bit between ring positions, so it is tabulated per position and indexed by the lock-step sample count. Fails when the ring
// would have fewer than 2 or more than max_size positions.
bool delay_table(double fractdelay, int max_size, std::vector<double> &w, int *k_out)
{
    const int size = (int)std::ceil(fractdelay) + 1;
    if (size > max_size || size < 2) return false;
    w.assign(size, 0.0);
    for (int bp = 0; bp < size; bp++) {
        double dptr = ((double)bp) - fractdelay;
        while (std::floor(dptr) < 0) dptr += ((double)size);
        const int iptr = (int)std::floor(dptr);
        w[bp] = dptr - ((double)iptr);
        // the shift-register form needs the read position to be "ceil(fd) samples ago" at every ring position
        int expect = bp - (int)std::ceil(fractdelay); while (expect < 0) expect += size;
        if (iptr != expect) return false;
    }
    *k_out = (int)std::ceil(fractdelay);
    return true;
}
// The OQPSK timing delays T/4 and T/8 ride in the kernel parameter block: at most 4 ring positions.
bool delay_table4(double fractdelay, double *w_out /*[4]*/, int *k_out)
{
    std::vector<double> w;
    if (!delay_table(fractdelay, 4, w, k_out)) return false;
    std::copy(w.begin(), w.end(), w_out);
    return true;
}

// W_n^k = exp(-2 pi i k / n), k = 0 .. n-1
std::vector<std::complex<double>> twiddles(int n)
{
    std::vector<std::complex<double>> tw(n);
    for (int k = 0; k < n; k++) { const double a = -2.0 * M_PI * (double)k / (double)n; tw[k] = std::complex<double>(cos(a), sin(a)); }
    return tw;
}
// In-place radix-2 FFT on the host (power-of-two length; tw = twiddles(H.size()))
void host_fft(std::vector<std::complex<double>> &H, const std::vector<std::complex<double>> &tw)
{
    const int NF = (int)H.size();
    int bits = 0; while ((1 << bits) < NF) bits++;
    for (int i = 0; i < NF; i++) { int r = 0; for (int q = 0; q < bits; q++) if (i & (1 << q)) r |= 1 << (bits - 1 - q); if (r > i) std::swap(H[i], H[r]); }
    for (int len = 2; len <= NF; len <<= 1)
        for (int i = 0; i < NF; i += len)
            for (int k = 0; k < len / 2; k++) { auto w = tw[k * (NF / len)]; auto u = H[i + k], v = H[i + k + len / 2] * w; H[i + k] = u + v; H[i + k + len / 2] = u - v; }
}

template <class T> int dev_alloc_zero(T **p, size_t count, cudaStream_t s)
{
    JB_CUDA(cudaMalloc((void **)p, count * sizeof(T)));
    JB_CUDA(cudaMemsetAsync(*p, 0, count * sizeof(T), s));
    return 0;
}
// A zeroed device buffer that lives as long as its owner: freed by release()
template <class O, class T> int owned_alloc(O *o, T **p, size_t count)
{
    int r = dev_alloc_zero(p, count, o->stream);
    if (r == 0) o->allocs.push_back((void *)*p);
    return r;
}
// Grow-on-demand device buffer of *cap elements. A buffer that is too small is replaced once `s` has drained, since queued
// work may still read it. `counts`, when given, is a companion buffer of n_counts ints that is replaced with it.
template <class T> int grow(T **buf, size_t *cap, size_t need, cudaStream_t s, int **counts = nullptr, size_t n_counts = 0)
{
    if (need <= *cap) return 0;
    JB_CUDA(cudaStreamSynchronize(s));
    cudaFree(*buf); *buf = 0;
    if (counts) { cudaFree(*counts); *counts = 0; }
    JB_CUDA(cudaMalloc(buf, need * sizeof(T)));
    if (counts) JB_CUDA(cudaMalloc(counts, n_counts * sizeof(int)));
    *cap = need;
    return 0;
}
// End of a destroy, after the family's own synchronisation: frees the owned buffers, the grow-on-demand buffers and pinned
// host mirrors listed, the stream and the object.
template <class O> void release(O *o, std::initializer_list<void *> grown, std::initializer_list<void *> pinned, cudaStream_t stream)
{
    for (void *q : o->allocs) cudaFree(q);
    for (void *q : grown) cudaFree(q);
    for (void *q : pinned) cudaFreeHost(q);
    if (stream) cudaStreamDestroy(stream);
    delete o;
}
// The trig tables exactly as TrigLookUp builds them (DSP.cpp:19-20), computed with the host libm, in two owned buffers.
// The copies read `host`, which the caller keeps alive until it synchronises the stream.
template <class O> int upload_wave_table(O *o, std::vector<double> &host, const double **sin_t, const double **cos_t)
{
    host.resize(2 * jb::WTSIZE);
    double *sn = host.data(), *cs = host.data() + jb::WTSIZE;
    for (int i = 0; i < jb::WTSIZE; i++) sn[i] = (sin(2 * M_PI * ((double)i) / jb::WTSIZE));
    for (int i = 0; i < jb::WTSIZE; i++) cs[i] = (sin(M_PI_2 + 2 * M_PI * ((double)i) / jb::WTSIZE));
    double *ds, *dc;
    if (owned_alloc(o, &ds, (size_t)jb::WTSIZE) || owned_alloc(o, &dc, (size_t)jb::WTSIZE)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(ds, sn, jb::WTSIZE * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaMemcpyAsync(dc, cs, jb::WTSIZE * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    *sin_t = ds; *cos_t = dc;
    return 0;
}

// JFastFir::setKernel for n_channels streams (fastfir.cuh): H = FFT of the zero-padded kernel `taps`, the twiddles, and zeroed
// history and staging rows, all owned by o
template <class O> int fastfir_create(O *o, const std::vector<std::complex<double>> &taps, int nfft, int n_channels, FastFir &f)
{
    memset(&f, 0, sizeof f);
    f.K = (int)taps.size(); f.nfft = nfft; f.L = nfft - f.K + 1;
    if (!fastfir_size_supported(f.K, nfft)) { set_error("internal: no FFT convolution kernel for this kernel length and nfft"); return JAERO_E_ARG; }
    std::vector<std::complex<double>> H(nfft, 0.0);
    std::copy(taps.begin(), taps.end(), H.begin());
    const std::vector<std::complex<double>> tw = twiddles(nfft);
    host_fft(H, tw);
    const size_t C = n_channels;
    if (owned_alloc(o, &f.H, (size_t)nfft) || owned_alloc(o, &f.tw, (size_t)nfft) || owned_alloc(o, &f.hist, C * (f.K - 1)) ||
        owned_alloc(o, &f.inblk, C * f.L) || owned_alloc(o, &f.outblk, C * f.L)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(f.H, H.data(), nfft * sizeof(double2), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaMemcpyAsync(f.tw, tw.data(), nfft * sizeof(double2), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaStreamSynchronize(o->stream));
    return 0;
}
// JFastFir::update over samples [0, n) of one call: exchange(i0, i1, fill0) launches the caller's exchange kernel for samples
// [i0, i1) at staging position fill0, and the block transform runs whenever the staging block fills. Counts its launches.
template <class X> int fastfir_feed(FastFir &f, int n, int n_channels, cudaStream_t s, long long *launches, X exchange)
{
    int i = 0;
    while (i < n) {
        const int take = std::min(f.L - f.fill, n - i);
        if (exchange(i, i + take, f.fill)) return JAERO_E_CUDA;
        (*launches)++;
        f.fill += take; i += take;
        if (f.fill == f.L) {
            if (fastfir_block_launch(f, n_channels, f.blocks == 0 ? 1 : 0, s)) return JAERO_E_CUDA;
            (*launches)++;
            f.fill = 0; f.blocks++;
        }
    }
    return 0;
}

// After a host read: move the not-yet-emitted (<32 / <12) soft bits to the front of each ring. soft_total (drained-value
// totals) and lost_n (SignalStatus(false) events, consumed by the frame layer before the ring is reset) may be null.
__global__ void soft_reset_kernel(int n_channels, int *count_col, const int *pending_col, int16_t *soft, int soft_cap,
                                  long long *soft_total, int *lost_n)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels) return;
    int &count = count_col[ch];
    const int pending = pending_col[ch];
    int16_t *ring = soft + (size_t)ch * soft_cap;
    for (int k = 0; k < pending; k++) ring[k] = ring[count + k];
    if (soft_total) soft_total[ch] += count;
    count = 0;
    if (lost_n) lost_n[ch] = 0;
}
// col[ch] = value for one channel, or for every channel when channel < 0
__global__ void set_int_kernel(int *col, int n_channels, int channel, int value)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n_channels) return;
    if (channel < 0 || channel == ch) col[ch] = value;
}
int launch_set_int(int *col, int n_channels, int channel, int value, cudaStream_t s)
{
    set_int_kernel<<<(n_channels + 127) / 128, 128, 0, s>>>(col, n_channels, channel, value);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int soft_reset(const DemodParams &p, cudaStream_t s)
{
    const size_t cp = p.cpad;
    soft_reset_kernel<<<(p.n_channels + 127) / 128, 128, 0, s>>>(p.n_channels, p.I + (size_t)I_SOFT_COUNT * cp, p.I + (size_t)I_SOFT_PENDING * cp,
                                                                  p.soft, p.soft_cap, p.soft_total, p.I + (size_t)I_LOST_N * cp);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int soft_reset(const BurstParams &p, cudaStream_t s)
{
    const size_t cp = p.cpad;
    soft_reset_kernel<<<(p.n_channels + 127) / 128, 128, 0, s>>>(p.n_channels, p.BI + (size_t)BI_SOFT_COUNT * cp, p.BI + (size_t)BI_SOFT_PENDING * cp,
                                                                  p.soft, p.soft_cap, nullptr, nullptr);
    JB_CUDA(cudaGetLastError());
    return 0;
}
// The soft-bit read-out of both demodulator families: pull the n_rows x cpad int block (soft-bit counts in row cnt_row,
// overflow flags in row ovf_row), refuse an overflow, copy the filled part of every ring out in one 2-D copy, unpack it per
// channel and reset the rings.
template <class P> int drain_softbits(const P &p, const int *d_ints, int n_rows, int cnt_row, int ovf_row, int *h_ints, int16_t *h_stage,
                                      cudaStream_t s, int16_t *out, size_t cap, int32_t *counts)
{
    const size_t cp = p.cpad;
    JB_CUDA(cudaMemcpyAsync(h_ints, d_ints, (size_t)n_rows * cp * sizeof(int), cudaMemcpyDeviceToHost, s));
    JB_CUDA(cudaStreamSynchronize(s));
    const int *cnt = h_ints + (size_t)cnt_row * cp, *ovf = h_ints + (size_t)ovf_row * cp;
    int maxc = 0; bool overflow = false;
    for (int ch = 0; ch < p.n_channels; ch++) { maxc = std::max(maxc, cnt[ch]); overflow |= (ovf[ch] != 0) || ((size_t)cnt[ch] > cap); }
    if (overflow) { set_error("soft-bit ring overflow: drain more often or pass a larger buffer"); return JAERO_E_OVERFLOW; }
    if (maxc > 0) {
        JB_CUDA(cudaMemcpy2DAsync(h_stage, (size_t)p.soft_cap * 2, p.soft, (size_t)p.soft_cap * 2, (size_t)maxc * 2, p.n_channels,
                                  cudaMemcpyDeviceToHost, s));
        JB_CUDA(cudaStreamSynchronize(s));
    }
    for (int ch = 0; ch < p.n_channels; ch++) {
        counts[ch] = cnt[ch];
        if (cnt[ch]) memcpy(out + (size_t)ch * cap, h_stage + (size_t)ch * p.soft_cap, (size_t)cnt[ch] * 2);
    }
    return soft_reset(p, s);
}
} // namespace

struct jaero_batch {
    jaero_settings set;
    int device;
    cudaStream_t stream;
    DemodParams p;
    CfePlan cfe;
    std::vector<void *> allocs;
    // lock-step counters mirrored on the host
    long long samples;          // samples fully processed
    int bb_pos, coarse_counter;
    int16_t *d_stage; size_t stage_cap;
    // 8400 bps pre-filter (K6)
    bool pre_on; PreParams pre; FastFir fir; double2 *d_x; size_t x_cap;
    int16_t *h_soft_stage;      // pinned
    int *h_ints; double *h_dbls; long long *h_soft_total;   // pinned mirrors of I / D / soft_total
    long long launches;
    cudaStream_t own_stream;
    bool profiling;
    // host-input pipelining (jaero_batch_write): the H2D copy is cut into column slices on a copy stream; a segment only
    // waits for the slices it reads
    cudaStream_t copy_stream; cudaEvent_t ev_slice[8], ev_stage_free; int n_slices, slice_len, next_slice;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_seg, ev_cfe;
    double prof_samples;
    // seating of the channels in the pipelined 10500 bps kernel (regroup)
    int *d_chan_of; double *d_keys, *h_keys; double *d_ring_scratch; size_t ring_scratch_count;
    std::vector<int> slot_of;   // [cpad] seat of channel c
    long long epochs, next_regroup;   // next_regroup: estimator epoch of the next seating check, -1 = never
};

namespace {
__global__ void init_state_kernel(DemodParams p, const double *freq_center, double st_freq, double ebno_init)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= p.n_channels) return;
    auto D = [&](int i) -> double & { return p.D[(size_t)i * p.cpad + ch]; };
    auto I = [&](int i) -> int & { return p.I[(size_t)i * p.cpad + ch]; };
    // WaveTable::SetFreq(double,int) (DSP.cpp:142-149): WTstep = freq*WTSIZE/(float)samplerate
    double fc = freq_center[ch];
    if (fc > ((p.Fs / 2.0) - (p.lockingbw / 2.0))) fc = ((p.Fs / 2.0) - (p.lockingbw / 2.0));   // oqpskdemodulator.cpp:183
    if (fc < 0) fc = 0;
    const double sr = (double)((float)((int)p.Fs));
    D(D_M2_FREQ) = fc; D(D_M2_STEP) = (fc) * ((double)jb::WTSIZE) / sr;
    D(D_MC_FREQ) = fc; D(D_MC_STEP) = (fc) * ((double)jb::WTSIZE) / sr;
    D(D_ST_FREQ) = st_freq; D(D_ST_STEP) = (st_freq) * ((double)jb::WTSIZE) / sr;
    D(D_SR_FREQ) = st_freq; D(D_SR_STEP) = (st_freq) * ((double)jb::WTSIZE) / sr;
    D(D_MSE) = (p.kind == JAERO_KIND_OQPSK) ? 100.0 : 10.0;       // oqpskdemodulator.cpp:17 / mskdemodulator.cpp:180
    D(D_DIFF_LAST) = -1.0;                                        // DSP.cpp:520
    D(D_EB_EBNO) = ebno_init;
    I(I_COUNTDOWN) = 4; I(I_COUNTDOWN2) = 5;                      // oqpskdemodulator.cpp:641,652 / mskdemodulator.cpp:493
    I(I_EMPTYING) = 1;                                            // coarsefreqestimate.cpp:24
}

// PeakVolume (oqpskdemodulator.cpp:393-405, mskdemodulator.cpp:329-344): max |sample| of the input since the last read-out.
// One warp per channel row, 16-byte loads; the same for every demodulator kernel variant.
__global__ void peak_kernel(DemodParams p, const int16_t *__restrict__ pcm, size_t stride, int n)
{
    const int ch = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (ch >= p.n_channels) return;
    const int4 *row = reinterpret_cast<const int4 *>(pcm + (size_t)ch * stride);
    int m = 0;
    for (int k = lane; k * 8 < n; k += 32) {
        const int4 v = __ldg(row + k);
        const int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int lo = (int)(short)(w[q] & 0xffff), hi = w[q] >> 16;
            if (k * 8 + 2 * q < n) m = max(m, abs(lo));
            if (k * 8 + 2 * q + 1 < n) m = max(m, abs(hi));
        }
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if (lane == 0) { int &pk = p.I[(size_t)I_PEAK * p.cpad + ch]; pk = max(pk, m); }
}
// CenterFreqChangedSlot (oqpskdemodulator.cpp:291-310 / mskdemodulator.cpp:265-282)
__global__ void center_freq_kernel(DemodParams p, int channel, double freq_center)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= p.n_channels || (channel >= 0 && channel != ch)) return;
    auto D = [&](int i) -> double & { return p.D[(size_t)i * p.cpad + ch]; };
    double fc = freq_center;
    if (p.kind == JAERO_KIND_OQPSK) {
        if (p.fb != 8400) { if (fc < (0.5 * p.fb)) fc = 0.5 * p.fb; if (fc > (p.Fs / 2.0 - 0.5 * p.fb)) fc = p.Fs / 2.0 - 0.5 * p.fb; }
    } else { if (fc < (0.75 * p.fb)) fc = 0.75 * p.fb; if (fc > (p.Fs / 2.0 - 0.75 * p.fb)) fc = p.Fs / 2.0 - 0.75 * p.fb; }
    if (fc < 0) fc = 0;
    const double srf = (double)((float)((int)p.Fs));
    D(D_MC_FREQ) = fc; D(D_MC_STEP) = (fc) * ((double)jb::WTSIZE) / srf;   // SetFreq(freq,Fs)
    auto set_m2 = [&](double f) { if (f < 0) f = 0; D(D_M2_FREQ) = f; D(D_M2_STEP) = (f) * ((double)jb::WTSIZE) / p.Fs; };
    if (p.afc) set_m2(D(D_MC_FREQ));
    if ((D(D_M2_FREQ) - D(D_MC_FREQ)) > (p.lockingbw / 2.0)) set_m2(D(D_MC_FREQ) + (p.lockingbw / 2.0));
    if ((D(D_M2_FREQ) - D(D_MC_FREQ)) < (-p.lockingbw / 2.0)) set_m2(D(D_MC_FREQ) - (p.lockingbw / 2.0));
    double2 *row = p.bb + (size_t)ch * p.bb_len;
    for (int j = 0; j < p.bb_len; j++) row[j] = make_double2(0.0, 0.0);
}
// ---- seating by symbol-timing phase (pipelined 10500 bps kernel)
static const int REGROUP_EVERY = 128;      // estimator epochs between seating checks after the first two (see jaero_batch_create)
static const double REGROUP_SPREAD = 1.5;  // samples of strobe-phase spread at which a CTA counts as drifted apart
// key[c] = samples until channel c's next carrier-update strobe, in [0, 2 * samples per strobe): st_osc passes the point ee
// (oqpskdemodulator.cpp:488) every Fs/fb samples and every second passage (yui, :496-503) is a carrier update.
__global__ void regroup_key_kernel(DemodParams p, double *__restrict__ key)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= p.n_channels) return;
    const double ptr = p.D[(size_t)D_ST_PTR * p.cpad + ch], step = p.D[(size_t)D_ST_STEP * p.cpad + ch];
    const int yui = p.I[(size_t)I_YUI * p.cpad + ch];
    const double N = (double)jb::WTSIZE;
    double d = p.ee * N - ptr; if (d < 0) d += N;
    const double per = step > 0 ? N / step : 1.0;
    double k = step > 0 ? d / step : 0.0;
    if (yui) k += per;                                    // the next passage only stores pt_d; the one after it updates the carrier
    key[ch] = fmod(k, 2.0 * per);
}
// ring_new[(cta', k, lane')] = ring_old[(cta, k, lane)] for the channel that moves from seat (cta, lane) to (cta', lane')
__global__ void regroup_ring_kernel(const double *__restrict__ src, double *__restrict__ dst, const int *__restrict__ old_seat_of_new, int len, int n_ctas)
{
    const int lane = threadIdx.x & 31;
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // (cta', k)
    if (row >= (long long)n_ctas * len) return;
    const int cta_n = (int)(row / len), k = (int)(row % len);
    const int so = old_seat_of_new[cta_n * 32 + lane];
    dst[row * 32 + lane] = src[((size_t)(so >> 5) * len + k) * 32 + (so & 31)];
}
// New seating: slot_of[c] for every channel (pads keep their seats). The rings follow; everything else is indexed by channel.
int batch_apply_seating(jaero_batch *b, const std::vector<int> &new_slot_of)
{
    DemodParams &p = b->p;
    const int cp = p.cpad, n_ctas = cp / 32;
    std::vector<int> old_seat_of_new(cp), chan_of(cp);
    for (int c = 0; c < cp; c++) { old_seat_of_new[new_slot_of[c]] = b->slot_of[c]; chan_of[new_slot_of[c]] = c; }
    const size_t need = (size_t)p.agc_len * cp;
    if (!b->d_ring_scratch) {
        if (cudaMalloc(&b->d_ring_scratch, need * sizeof(double)) != cudaSuccess) { cudaGetLastError(); b->next_regroup = -1; return 0; }   // no room: keep the seating
        b->ring_scratch_count = need;
    }
    int *d_map = b->d_chan_of + cp;                          // second half of the allocation: old seat of each new seat
    JB_CUDA(cudaMemcpyAsync(d_map, old_seat_of_new.data(), cp * sizeof(int), cudaMemcpyHostToDevice, b->stream));
    auto move = [&](double *ring, int len) -> int {
        if (!ring) return 0;
        const long long rows = (long long)n_ctas * len;
        regroup_ring_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, b->stream>>>(ring, b->d_ring_scratch, d_map, len, n_ctas);
        JB_CUDA(cudaGetLastError());
        JB_CUDA(cudaMemcpyAsync(ring, b->d_ring_scratch, (size_t)rows * 32 * sizeof(double), cudaMemcpyDeviceToDevice, b->stream));
        b->launches++;
        return 0;
    };
    if (move(p.agc_ring, p.agc_len) || move(p.ebno_e1, p.ebno_len) || move(p.ebno_e2, p.ebno_len)) return -1;
    JB_CUDA(cudaMemcpyAsync(b->d_chan_of, chan_of.data(), cp * sizeof(int), cudaMemcpyHostToDevice, b->stream));
    JB_CUDA(cudaStreamSynchronize(b->stream));               // the host vectors above go out of scope
    b->slot_of = new_slot_of;
    return 0;
}
int batch_regroup_by_phase(jaero_batch *b, bool force)
{
    DemodParams &p = b->p;
    const int C = p.n_channels, cp = p.cpad;
    regroup_key_kernel<<<(C + 127) / 128, 128, 0, b->stream>>>(p, b->d_keys);
    JB_CUDA(cudaGetLastError());
    JB_CUDA(cudaMemcpyAsync(b->h_keys, b->d_keys, C * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    JB_CUDA(cudaStreamSynchronize(b->stream));
    b->launches++;
    // Is the present seating still coherent? A CTA is coherent when the carrier-update strobes of its channels fall within 1.5
    // samples of each other (circularly, period = two strobe intervals). Moving the rings costs ~30 ms per 4096 channels, so the
    // seating is only changed when more than a quarter of the CTAs have drifted apart (never, for transmitters on one clock).
    if (!force) {
        const double period = 2.0 * p.Fs / p.fb;                                     // keys are in [0, 2*Fs/fb)
        int bad = 0, ctas = 0;
        std::vector<double> ks;
        std::vector<std::vector<int>> members(cp / 32);
        for (int c = 0; c < C; c++) members[b->slot_of[c] >> 5].push_back(c);
        for (auto &m : members) {
            if (m.size() < 2) continue;
            ctas++;
            ks.clear();
            for (int c : m) ks.push_back(b->h_keys[c]);
            std::sort(ks.begin(), ks.end());
            double gap = ks.front() + period - ks.back();
            for (size_t i = 1; i < ks.size(); i++) gap = std::max(gap, ks[i] - ks[i - 1]);
            if (period - gap > REGROUP_SPREAD) bad++;
        }
        if (bad * 4 <= ctas) return 0;
    }
    std::vector<int> order(C);
    for (int c = 0; c < C; c++) order[c] = c;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return b->h_keys[x] < b->h_keys[y]; });
    std::vector<int> slot_of(cp);
    for (int k = 0; k < C; k++) slot_of[order[k]] = k;
    for (int c = C; c < cp; c++) slot_of[c] = c;
    if (slot_of == b->slot_of) return 0;
    return batch_apply_seating(b, slot_of);
}
} // namespace

extern "C" {

int jaero_batch_create(const jaero_settings *s, int n_channels, const double *freq_center_per_channel, int device, jaero_batch **out)
{
    if (!s || !out || n_channels <= 0) { set_error("jaero_batch_create: bad argument"); return JAERO_E_ARG; }
    if (s->kind != JAERO_KIND_OQPSK && s->kind != JAERO_KIND_MSK) { set_error("jaero_batch_create: unknown kind"); return JAERO_E_ARG; }
    if (s->Fs <= 0 || s->fb <= 0 || s->coarsefreqest_fft_power < 10 || s->coarsefreqest_fft_power > 14) {
        set_error("jaero_batch_create: Fs/fb must be positive and coarsefreqest_fft_power in 10..14"); return JAERO_E_ARG; }
    CreateGuard<jaero_batch> guard(jaero_batch_destroy);
    { int r = guard.begin("jaero_batch_create", device); if (r) return r; }
    jaero_batch *b = guard.obj;
    b->set = *s; b->samples = 0; b->bb_pos = 0; b->coarse_counter = 0;
    b->d_stage = 0; b->stage_cap = 0; b->launches = 0;
    b->pre_on = false; b->d_x = 0; b->x_cap = 0;
    b->own_stream = b->stream; b->profiling = false; b->prof_samples = 0;
    b->copy_stream = 0; b->ev_stage_free = 0; for (int k = 0; k < 8; k++) b->ev_slice[k] = 0; b->n_slices = 0; b->slice_len = 0; b->next_slice = 0;
    DemodParams &p = b->p;
    memset(&p, 0, sizeof p);
    p.kind = s->kind; p.n_channels = n_channels; p.cpad = (n_channels + 31) & ~31;
    p.Fs = s->Fs; p.fb = s->fb; p.lockingbw = s->lockingbw; p.signalthreshold = s->signalthreshold;
    p.afc = s->afc; p.sql = s->sql; p.cpu_reduce = s->cpu_reduce; p.report_ebno = s->report_ebno;
    p.bbnfft = 1 << s->coarsefreqest_fft_power;
    p.bb_len = p.bbnfft;
    std::vector<double> taps;
    double st_freq;
    if (s->kind == JAERO_KIND_OQPSK) {
        taps = (s->fb == 8400) ? rrc_taps(0.6, 55, s->Fs, s->fb / 2) : rrc_taps(1.0, 55, s->Fs, s->fb / 2);   // oqpskdemodulator.cpp:209-211
        p.agc_len = (int)round(4 * s->Fs);                                    // :197 AGC(4,Fs)
        p.ebno_len = 2 * 48000;                                               // :42 (built in the ctor with Fs=48000)
        p.marg_len = 800; p.dt_len = 401; p.mse_len = 400;                    // :44-45,53
        const double T = s->Fs / (s->fb / 2);                                 // :221
        if (!delay_table4(T / 4.0, p.w41v, &p.k41) || !delay_table4(T / 8.0, p.w8v, &p.k8)) {
            set_error("unsupported fractional delay for this Fs/fb"); return JAERO_E_ARG; }
        if (s->fb == 8400) {                                                  // :243-250 (the 10 Hz set, assigned last, wins)
            p.res_b0 = 0.0012845857864470789; p.res_b1 = 0; p.res_b2 = -0.0012845857864470789;
            p.res_a1 = -0.90681461999279889; p.res_a2 = 0.99743082842710584;
            p.ee = 0.65;
        } else {
            p.res_b0 = 0.00032714218939589035; p.res_b1 = 0; p.res_b2 = 0.00032714218939589035;   // :256-261
            p.res_a1 = -0.39005299948210803; p.res_a2 = 0.99934571562120822;
            p.ee = 0.4;                                                       // :263
        }
        p.lf_b0 = 0.0010275610653672064; p.lf_b1 = 0.0020551221307344128; p.lf_b2 = 0.0010275610653672064;   // :95-100
        p.lf_a1 = -1.9207386815577139; p.lf_a2 = 0.92509247310306331;
        st_freq = s->fb;                                                      // :270
    } else {
        p.sps = (int)(s->Fs / s->fb);                                         // mskdemodulator.cpp:149
        if (2 * p.sps > MAX_TAPS) { set_error("MSK: 2*SamplesPerSymbol exceeds the supported FIR length"); return JAERO_E_ARG; }
        taps.resize(2 * p.sps);
        for (int i = 0; i < 2 * p.sps; i++) taps[i] = sin(M_PI * i / (2.0 * p.sps)) / (2.0 * p.sps);   // :164-170
        p.agc_len = (int)round(1 * s->Fs);                                    // :173
        p.ebno_len = (int)(2.0 * s->Fs);                                      // :176
        p.marg_len = p.sps; p.dt_len = p.sps / 2 + 1; p.mse_len = 600;        // :254-256, ctor :64
        if (s->fb >= 1200) {                                                  // :189-250
            p.correctionfactor = 0.6;
            if (s->Fs == 48000) { p.res_a1 = -1.993312819378528; p.res_a2 = 0.999476538254407; p.res_b0 = 2.617308727964618e-04; p.res_b2 = -2.617308727964618e-04; p.ee = 0.025; }
            else { p.res_a1 = -1.974342917561558; p.res_a2 = 0.998953350377616; p.res_b0 = 5.233248111921052e-04; p.res_b2 = -5.233248111921052e-04; p.ee = 0.05; }
        } else {
            p.correctionfactor = 1.0;
            if (s->Fs == 48000) { p.res_a1 = -1.998196509168551; p.res_a2 = 0.999738234875681; p.res_b0 = 1.308825621597620e-04; p.res_b2 = -1.308825621597620e-04; p.ee = 0.025; }
            else { p.res_a1 = -1.974342917561558; p.res_a2 = 0.998953350377616; p.res_b0 = 5.233248111921052e-04; p.res_b2 = -5.233248111921052e-04; p.ee = 0.0125; }
        }
        p.res_b1 = 0;
        st_freq = s->fb / 2;                                                  // :159
    }
    if ((p.agc_len % 32) || (p.ebno_len % 32) || p.agc_len < 96 || p.ebno_len < 96) {
        set_error("unsupported sample rate: the AGC / EbNo window lengths must be multiples of 32 samples"); return JAERO_E_ARG; }
    p.ntaps = (int)taps.size();
    p.soft_cap = std::max(4096, (int)(2 * s->fb) + 64);
    if (p.ntaps > MAX_TAPS) { set_error("too many FIR taps"); return JAERO_E_ARG; }
    for (int k = 0; k < p.ntaps; k++) p.taps[k] = taps[k];   // per-batch: the taps ride in the kernel parameter block

    const size_t cp = p.cpad;
    int rc = 0;
    rc |= owned_alloc(b, &p.D, (size_t)D_COUNT * cp);
    rc |= owned_alloc(b, &p.I, (size_t)I_COUNT * cp);
    rc |= owned_alloc(b, &p.agc_ring, (size_t)p.agc_len * cp);
    if (p.report_ebno) { rc |= owned_alloc(b, &p.ebno_e1, (size_t)p.ebno_len * cp); rc |= owned_alloc(b, &p.ebno_e2, (size_t)p.ebno_len * cp); }
    rc |= owned_alloc(b, &p.fir_re, (size_t)(p.ntaps + 1) * cp);
    rc |= owned_alloc(b, &p.fir_im, (size_t)(p.ntaps + 1) * cp);
    rc |= owned_alloc(b, &p.bb, (size_t)n_channels * p.bb_len);
    rc |= owned_alloc(b, &p.marg_ring, (size_t)p.marg_len * cp);
    rc |= owned_alloc(b, &p.mse_pm, (size_t)p.mse_len * cp);
    rc |= owned_alloc(b, &p.mse_ma, (size_t)p.mse_len * cp);
    rc |= owned_alloc(b, &p.dt_ring, (size_t)p.dt_len * cp);
    if (s->kind == JAERO_KIND_MSK) {
        rc |= owned_alloc(b, &p.dsmpl_ring, (size_t)(p.sps + 1) * cp);
        rc |= owned_alloc(b, &p.dly8_ring, (size_t)(p.sps / 2 + 1) * cp);
    }
    rc |= owned_alloc(b, &p.soft, (size_t)n_channels * p.soft_cap);
    rc |= owned_alloc(b, &p.soft_total, (size_t)cp);
    rc |= owned_alloc(b, &p.lost_pos, (size_t)LOST_CAP * cp);
    rc |= owned_alloc(b, &p.cfe_est_out, (size_t)cp);
    if (rc) return JAERO_E_CUDA;

    {
        std::vector<double> wt;
        if (upload_wave_table(b, wt, &p.sin_t, &p.cos_t)) return JAERO_E_CUDA;
        JB_CUDA(cudaStreamSynchronize(b->stream));
    }
    // coarse estimator plan (CoarseFreqEstimate::setSettings, coarsefreqestimate.cpp:39-76)
    {
        CfePlan &c = b->cfe;
        memset(&c, 0, sizeof c);
        c.nfft = p.bbnfft;
        const int lg = s->coarsefreqest_fft_power;
        c.n1 = 1 << ((lg + 1) / 2); c.n2 = 1 << (lg / 2);
        c.hzperbin = s->Fs / ((double)c.nfft);
        const double lbw = (s->kind == JAERO_KIND_OQPSK) ? 2.0 * s->lockingbw / 2.0 : s->lockingbw;   // oqpskdemodulator.cpp:191
        c.startbin = (int)std::max(round(lbw / c.hzperbin), 1.0);
        c.stopbin = c.nfft - c.startbin;
        c.expectedpeakbin = (int)round(s->fb / (2.0 * c.hzperbin));
        c.lo = (int)round((-lbw / c.hzperbin) + ((double)(c.nfft / 2)));
        c.hi = (int)round((lbw / c.hzperbin) + ((double)(c.nfft / 2)));
        c.is8400 = (s->fb == 8400);
        const std::vector<std::complex<double>> tw = twiddles(c.nfft);
        // channels per pass group: the two work buffers of a group (2 x group x nfft x 16 B) (larger groups amortise launch tails)
        c.group = std::min(n_channels, 1024);
        if (c.nfft == 16384) c.clusters = cfe_cluster_capacity();
        if (owned_alloc(b, &c.tw, (size_t)c.nfft) || owned_alloc(b, &c.work_a, (size_t)c.group * c.nfft) ||
            owned_alloc(b, &c.work_b, (size_t)c.group * c.nfft) || owned_alloc(b, &c.y, (size_t)n_channels * c.nfft)) return JAERO_E_CUDA;
        JB_CUDA(cudaMemcpyAsync(c.tw, tw.data(), tw.size() * sizeof(double2), cudaMemcpyHostToDevice, b->stream));
        if (c.is8400) {                                                       // raised-cosine window (coarsefreqestimate.cpp:62-74)
            std::vector<double> win(c.nfft, 0.0);
            win[0] = 1;
            for (int i = 1; i <= c.startbin; i++) {
                double val = cos(M_PI_2 * ((double)i) / ((double)c.startbin)); val *= val;
                if ((c.nfft - i) < 0) break;
                if (i >= c.nfft) break;
                win[c.nfft - i] = val; win[i] = val;
            }
            if (owned_alloc(b, &c.window, (size_t)c.nfft)) return JAERO_E_CUDA;
            JB_CUDA(cudaMemcpyAsync(c.window, win.data(), win.size() * sizeof(double), cudaMemcpyHostToDevice, b->stream));
        }
        JB_CUDA(cudaStreamSynchronize(b->stream));
    }
    if (s->kind == JAERO_KIND_OQPSK && s->fb == 8400) {
        // K6: 2049-tap RRC (alpha 0.6) applied by streaming FFT convolution, nfft 4096 (oqpskdemodulator.cpp:280-283)
        b->pre_on = true;
        const std::vector<double> kern = rrc_taps(0.6, 2048, s->Fs, s->fb / 2);
        { int r = fastfir_create(b, std::vector<std::complex<double>>(kern.begin(), kern.end()), 4096, n_channels, b->fir); if (r) return r; }
        PreParams &q = b->pre; memset(&q, 0, sizeof q);
        if (owned_alloc(b, &q.osc, (size_t)4 * cp) || owned_alloc(b, &p.m2_freq_sum, (size_t)cp)) return JAERO_E_CUDA;
        // mixer_fir_pre.SetFreq(freq_center,Fs) is only done in the ctor, with the ctor's 8000 Hz (oqpskdemodulator.cpp:21,115)
        std::vector<double> osc(4 * cp, 0.0);
        for (size_t c2 = 0; c2 < cp; c2++) { osc[1 * cp + c2] = (8000.0) * ((double)jb::WTSIZE) / ((double)((float)48000)); osc[2 * cp + c2] = 8000.0; }
        JB_CUDA(cudaMemcpyAsync(q.osc, osc.data(), osc.size() * sizeof(double), cudaMemcpyHostToDevice, b->stream));
        JB_CUDA(cudaStreamSynchronize(b->stream));
        q.n_channels = n_channels; q.cpad = p.cpad; q.sin_t = p.sin_t; q.cos_t = p.cos_t;
    }
    // per-channel initial state
    {
        std::vector<double> fc(n_channels);
        for (int i = 0; i < n_channels; i++) fc[i] = freq_center_per_channel ? freq_center_per_channel[i] : s->freq_center;
        double *dfc;
        JB_CUDA(cudaMalloc(&dfc, n_channels * sizeof(double)));
        JB_CUDA(cudaMemcpyAsync(dfc, fc.data(), n_channels * sizeof(double), cudaMemcpyHostToDevice, b->stream));
        init_state_kernel<<<(n_channels + 127) / 128, 128, 0, b->stream>>>(p, dfc, st_freq, 0.0);
        JB_CUDA(cudaGetLastError());
        JB_CUDA(cudaStreamSynchronize(b->stream));
        cudaFree(dfc);
    }
    b->d_chan_of = 0; b->d_keys = 0; b->h_keys = 0; b->d_ring_scratch = 0; b->ring_scratch_count = 0; b->epochs = 0;
    b->next_regroup = -1;
    if (s->kind == JAERO_KIND_OQPSK && s->fb > 8400 && !s->cpu_reduce) {
        // the pipelined kernel seats channels by symbol-timing phase: first after 2.9 s of signal (the timing loops' phases are final
        // to a few hundredths of a sample by then; at 2 s they are not), a check 2.7 s later (a no-op unless they moved),
        // then every REGROUP_EVERY estimator epochs (11 s: symbol clocks of different transmitters drift by a sample in minutes,
        // not seconds)
        if (owned_alloc(b, &b->d_chan_of, (size_t)2 * cp) || owned_alloc(b, &b->d_keys, (size_t)cp)) return JAERO_E_CUDA;
        JB_CUDA(cudaMallocHost(&b->h_keys, cp * sizeof(double)));
        b->slot_of.resize(cp);
        std::vector<int> ident(cp);
        for (size_t c = 0; c < cp; c++) { ident[c] = (int)c; b->slot_of[c] = (int)c; }
        JB_CUDA(cudaMemcpy(b->d_chan_of, ident.data(), cp * sizeof(int), cudaMemcpyHostToDevice));
        p.chan_of = b->d_chan_of;
        b->next_regroup = 34;
    }
    JB_CUDA(cudaMallocHost(&b->h_ints, (size_t)I_COUNT * cp * sizeof(int)));
    JB_CUDA(cudaMallocHost(&b->h_dbls, (size_t)D_COUNT * cp * sizeof(double)));
    JB_CUDA(cudaMallocHost(&b->h_soft_total, cp * sizeof(long long)));
    JB_CUDA(cudaMallocHost(&b->h_soft_stage, (size_t)n_channels * p.soft_cap * sizeof(int16_t)));
    guard.release();
    *out = b;
    return JAERO_OK;
}

void jaero_batch_destroy(jaero_batch *b)
{
    if (!b) return;
    cudaSetDevice(b->device);
    cudaStreamSynchronize(b->stream);
    if (b->copy_stream) { cudaStreamSynchronize(b->copy_stream); cudaStreamDestroy(b->copy_stream); }
    if (b->ev_stage_free) cudaEventDestroy(b->ev_stage_free);
    for (int k = 0; k < 8; k++) if (b->ev_slice[k]) cudaEventDestroy(b->ev_slice[k]);
    for (auto &e : b->ev_seg) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    for (auto &e : b->ev_cfe) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    release(b, {b->d_stage, b->d_x, b->d_ring_scratch}, {b->h_ints, b->h_dbls, b->h_soft_stage, b->h_soft_total, b->h_keys}, b->own_stream);
}
int jaero_batch_channels(const jaero_batch *b) { return b ? b->p.n_channels : 0; }
int64_t jaero_batch_launch_count(const jaero_batch *b) { return b ? b->launches : 0; }

int jaero_batch_set_stream(jaero_batch *b, void *cuda_stream) { return switch_stream(b, cuda_stream); }
int jaero_batch_set_profiling(jaero_batch *b, int enabled)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->profiling = enabled != 0;
    return JAERO_OK;
}
int jaero_batch_get_profile(jaero_batch *b, double out[5])
{
    if (!b || !out) { set_error("null argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    JB_CUDA(cudaStreamSynchronize(b->stream));
    double seg = 0, cfe = 0;
    for (auto &e : b->ev_seg) { float ms = 0; cudaEventElapsedTime(&ms, e.first, e.second); seg += ms; cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    for (auto &e : b->ev_cfe) { float ms = 0; cudaEventElapsedTime(&ms, e.first, e.second); cfe += ms; cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    out[0] = seg; out[1] = (double)b->ev_seg.size(); out[2] = cfe; out[3] = (double)b->ev_cfe.size(); out[4] = b->prof_samples;
    b->ev_seg.clear(); b->ev_cfe.clear(); b->prof_samples = 0;
    return JAERO_OK;
}
int jaero_batch_cfe_clusters(const jaero_batch *b) { return b ? b->cfe.clusters : 0; }

// ---- test support: one coarse-estimator epoch on a caller-supplied ring (not part of the drop-in surface)
int jaero_batch_cfe_geometry(const jaero_batch *b, int32_t out[6])
{
    if (!b || !out) { set_error("jaero_batch_cfe_geometry: null argument"); return JAERO_E_ARG; }
    const CfePlan &c = b->cfe;
    out[0] = c.nfft; out[1] = b->p.bb_len; out[2] = c.lo; out[3] = c.hi; out[4] = c.expectedpeakbin; out[5] = c.clusters;
    return JAERO_OK;
}
int jaero_batch_probe_cfe(jaero_batch *b, const double *ring, int oldest, const int32_t *bigchange, int impl, int max_clusters,
                          int max_group, double *y_out, double *raw_est, double *emitted_est)
{
    if (!b || !ring) { set_error("jaero_batch_probe_cfe: null argument"); return JAERO_E_ARG; }
    DemodParams &p = b->p;
    const int C = p.n_channels, N = b->cfe.nfft;
    const size_t cp = p.cpad;
    if (oldest < 0 || oldest >= p.bb_len) { set_error("jaero_batch_probe_cfe: oldest outside the ring"); return JAERO_E_ARG; }
    if (impl < 0 || impl > 2 || max_clusters < 0 || max_group < 0) {
        set_error("jaero_batch_probe_cfe: bad impl / max_clusters / max_group"); return JAERO_E_ARG; }
    CfePlan plan = b->cfe;                                         // a smaller group runs on a prefix of the work buffers
    if (max_group > 0) plan.group = std::min(plan.group, max_group);
    JB_CUDA(cudaSetDevice(b->device));
    int clusters = b->cfe.clusters;                                // impl 0: the path jaero_batch_write takes
    if (impl == 1) clusters = 0;
    if (impl == 2) {
        clusters = (N == 16384) ? cfe_cluster_capacity() : 0;
        if (clusters <= 0) { set_error("jaero_batch_probe_cfe: the cluster estimator is not available for this batch / device"); return JAERO_E_STATE; }
    }
    if (clusters > 0 && max_clusters > 0) clusters = std::min(clusters, max_clusters);
    // the batch is idle before its state is touched
    JB_CUDA(cudaStreamSynchronize(b->stream));
    // Every copy is stream-ordered on b->stream (the estimator kernels' stream): a cudaMemcpy from pageable memory may return
    // before its DMA has landed, and b->stream does not synchronise with the legacy default stream. The host buffers the copies
    // read stay alive until the final cudaStreamSynchronize.
    const cudaStream_t s = b->stream;
    std::vector<int> em, zb;
    JB_CUDA(cudaMemcpyAsync(p.bb, ring, (size_t)C * p.bb_len * sizeof(double2), cudaMemcpyHostToDevice, s));
    if (bigchange) {                                               // what the demodulator kernels do on CoarseFreqEstimate::bigchange()
        em.resize(C); zb.resize(C);
        JB_CUDA(cudaMemcpyAsync(em.data(), p.I + (size_t)I_EMPTYING * cp, C * sizeof(int), cudaMemcpyDeviceToHost, s));
        JB_CUDA(cudaMemcpyAsync(zb.data(), p.I + (size_t)I_ZERO_BB * cp, C * sizeof(int), cudaMemcpyDeviceToHost, s));
        JB_CUDA(cudaStreamSynchronize(s));
        for (int c = 0; c < C; c++) if (bigchange[c]) { em[c] = 4; zb[c] = 1; }
        JB_CUDA(cudaMemcpyAsync(p.I + (size_t)I_EMPTYING * cp, em.data(), C * sizeof(int), cudaMemcpyHostToDevice, s));
        JB_CUDA(cudaMemcpyAsync(p.I + (size_t)I_ZERO_BB * cp, zb.data(), C * sizeof(int), cudaMemcpyHostToDevice, s));
    }
    if (clusters > 0 ? cfe_cluster_run(plan, p, oldest, std::min(clusters, C), s, &b->launches)
                     : cfe_run(plan, p, oldest, s, &b->launches)) return JAERO_E_CUDA;
    if (y_out) JB_CUDA(cudaMemcpyAsync(y_out, b->cfe.y, (size_t)C * N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (raw_est) JB_CUDA(cudaMemcpyAsync(raw_est, p.D + (size_t)D_CFE_EST * cp, C * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (emitted_est) JB_CUDA(cudaMemcpyAsync(emitted_est, p.cfe_est_out, C * sizeof(double), cudaMemcpyDeviceToHost, s));
    JB_CUDA(cudaStreamSynchronize(s));
    return JAERO_OK;
}

} // extern "C"

// ---- test support: kernels on caller data (not part of the drop-in surface)
namespace {
struct Probe {
    int device; cudaStream_t stream;
    std::vector<void *> allocs;
};
void probe_destroy(Probe *o)
{
    cudaSetDevice(o->device);
    if (o->stream) cudaStreamSynchronize(o->stream);
    release(o, {}, {}, o->stream);
}
} // namespace

extern "C" {

int jaero_probe_fastfir(int device, int nfft, const double *taps, int K, int n_channels, const double *x, size_t n,
                        const int32_t *writes, int n_writes, double *y)
{
    if (!taps || !x || !writes || !y || n_channels <= 0 || n_writes <= 0 || n == 0 || n > 0x7fffffff) {
        set_error("jaero_probe_fastfir: null argument or bad n_channels / n / n_writes"); return JAERO_E_ARG; }
    if (!fastfir_size_supported(K, nfft)) {
        set_error("jaero_probe_fastfir: no FFT convolution kernel for " + std::to_string(K) + " taps at nfft " + std::to_string(nfft));
        return JAERO_E_ARG;
    }
    long long total = 0;
    for (int w = 0; w < n_writes; w++) {
        if (writes[w] <= 0) { set_error("jaero_probe_fastfir: write " + std::to_string(w) + " has size <= 0"); return JAERO_E_ARG; }
        total += writes[w];
    }
    if (total != (long long)n) {
        set_error("jaero_probe_fastfir: the write sizes add up to " + std::to_string(total) + ", not n = " + std::to_string(n));
        return JAERO_E_ARG;
    }
    CreateGuard<Probe> guard(probe_destroy);                 // frees the buffers and the stream on every return
    { int r = guard.begin("jaero_probe_fastfir", device); if (r) return r; }
    Probe *o = guard.obj;
    std::vector<std::complex<double>> h(K);
    for (int k = 0; k < K; k++) h[k] = std::complex<double>(taps[2 * k], taps[2 * k + 1]);
    FastFir f;
    { int r = fastfir_create(o, h, nfft, n_channels, f); if (r) return r; }
    const size_t C = n_channels;
    double2 *dx = 0, *dy = 0;
    if (owned_alloc(o, &dx, C * n) || owned_alloc(o, &dy, C * n)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(dx, x, C * n * sizeof(double2), cudaMemcpyHostToDevice, o->stream));
    long long launches = 0;
    int pos = 0;
    for (int w = 0; w < n_writes; w++) {                      // one fastfir_feed per write, as a filter's write call runs it
        if (fastfir_feed(f, writes[w], n_channels, o->stream, &launches, [&](int i0, int i1, int fill0) {
                return fastfir_probe_exchange_launch(f, n_channels, dx, dy, n, pos + i0, pos + i1, fill0, o->stream); }))
            return JAERO_E_CUDA;
        pos += writes[w];
    }
    JB_CUDA(cudaMemcpyAsync(y, dy, C * n * sizeof(double2), cudaMemcpyDeviceToHost, o->stream));
    JB_CUDA(cudaStreamSynchronize(o->stream));
    return JAERO_OK;
}

int jaero_probe_math(int device, int op, size_t n, const double *a, const double *b, double *out)
{
    const bool two = op == JAERO_MATH_DIV_EXACT || op == JAERO_MATH_DIV_FAST || op == JAERO_MATH_ATAN2_FAST || op == JAERO_MATH_HYPOT_FAST ||
                     op == JAERO_MATH_DIV_FAST_CFE;
    if (op < JAERO_MATH_DIV_EXACT || op > JAERO_MATH_DIV_FAST_CFE) { set_error("jaero_probe_math: unknown op " + std::to_string(op)); return JAERO_E_ARG; }
    if (!a || !out || (two && !b) || n == 0) { set_error("jaero_probe_math: null argument or n == 0"); return JAERO_E_ARG; }
    CreateGuard<Probe> guard(probe_destroy);
    { int r = guard.begin("jaero_probe_math", device); if (r) return r; }
    Probe *o = guard.obj;
    double *da = 0, *db = 0, *dout = 0;
    if (owned_alloc(o, &da, n) || owned_alloc(o, &dout, n) || (two && owned_alloc(o, &db, n))) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(da, a, n * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    if (two) JB_CUDA(cudaMemcpyAsync(db, b, n * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    const bool cfe = op == JAERO_MATH_LOG10_GE1 || op == JAERO_MATH_DIV_FAST_CFE;
    if ((cfe ? probe_math_cfe_launch : probe_math_launch)(op, n, da, db, dout, o->stream)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(out, dout, n * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    JB_CUDA(cudaStreamSynchronize(o->stream));
    return JAERO_OK;
}

int jaero_probe_osc(int device, int n_lanes, int n_ops, const int32_t *op, const double *arg, double samplerate, double *log)
{
    if (!op || !arg || !log || n_lanes <= 0 || n_ops <= 0) { set_error("jaero_probe_osc: null argument or bad n_lanes / n_ops"); return JAERO_E_ARG; }
    if (!(samplerate > 0)) { set_error("jaero_probe_osc: samplerate must be positive"); return JAERO_E_ARG; }
    const size_t n = (size_t)n_lanes * n_ops;
    for (size_t e = 0; e < n; e++)
        if (op[e] < JAERO_OSC_SET_FREQ || op[e] > JAERO_OSC_SET_FREQ_SR) {
            set_error("jaero_probe_osc: unknown op " + std::to_string(op[e]) + " at " + std::to_string(e)); return JAERO_E_ARG; }
    CreateGuard<Probe> guard(probe_destroy);
    { int r = guard.begin("jaero_probe_osc", device); if (r) return r; }
    Probe *o = guard.obj;
    int32_t *dop = 0; double *darg = 0, *dlog = 0;
    if (owned_alloc(o, &dop, n) || owned_alloc(o, &darg, n) || owned_alloc(o, &dlog, 7 * n)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(dop, op, n * sizeof(int32_t), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaMemcpyAsync(darg, arg, n * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    if (probe_osc_launch(n_lanes, n_ops, dop, darg, samplerate, dlog, o->stream)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(log, dlog, 7 * n * sizeof(double), cudaMemcpyDeviceToHost, o->stream));
    JB_CUDA(cudaStreamSynchronize(o->stream));
    return JAERO_OK;
}

int jaero_batch_sync(jaero_batch *b) { return sync_stream(b); }

int jaero_batch_write_device(jaero_batch *b, const int16_t *d_pcm, size_t n, size_t stride)
{
    if (!b || !d_pcm) { set_error("jaero_batch_write_device: null argument"); return JAERO_E_ARG; }
    if (n == 0) return JAERO_OK;                                   // `if(!len)return 0;` oqpskdemodulator.cpp:337
    if (stride < n || n > 0x7fffffff) { set_error("jaero_batch_write_device: bad stride / length"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    const DemodParams &p = b->p;
    if ((((uintptr_t)d_pcm) & 15) || (stride & 7)) {
        // the kernels stage PCM rows with 16-byte bulk copies: re-pitch unaligned caller buffers on the device
        const size_t C = p.n_channels, pitch = (n + 7) & ~(size_t)7;
        if (d_pcm == b->d_stage) { set_error("internal: staging buffer misaligned"); return JAERO_E_STATE; }
        if (grow(&b->d_stage, &b->stage_cap, C * pitch, b->stream)) return JAERO_E_CUDA;
        JB_CUDA(cudaMemcpy2DAsync(b->d_stage, pitch * sizeof(int16_t), d_pcm, stride * sizeof(int16_t), n * sizeof(int16_t), C,
                                  cudaMemcpyDeviceToDevice, b->stream));
        d_pcm = b->d_stage; stride = pitch;
    }
    if (b->pre_on) {
        while (b->next_slice < b->n_slices) { JB_CUDA(cudaStreamWaitEvent(b->stream, b->ev_slice[b->next_slice], 0)); b->next_slice++; }
        // K6 over the whole call first (oqpskdemodulator.cpp:343-381), then the per-sample loop consumes its output
        const size_t C = p.n_channels, xs = (n + 7) & ~(size_t)7;
        if (grow(&b->d_x, &b->x_cap, C * xs, b->stream)) return JAERO_E_CUDA;
        b->pre.x = b->d_x; b->pre.xstride = xs;
        b->p.xpre = b->d_x; b->p.xstride = xs;
        if (pre_down_launch(b->pre, d_pcm, stride, (int)n, b->stream)) return JAERO_E_CUDA;
        b->launches++;
        if (fastfir_feed(b->fir, (int)n, p.n_channels, b->stream, &b->launches,
                         [&](int i0, int i1, int fill0) { return fir_exchange_up_launch(b->pre, b->fir, i0, i1, fill0, b->stream); }))
            return JAERO_E_CUDA;
    }
    const int N = p.bbnfft, trig_every = p.cpu_reduce ? N : N / 4;
    SegmentArgs a;
    memset(&a, 0, sizeof a);
    a.new_write = 1;
    int seg_start = 0; bool resume = false;
    auto launch = [&](int i0, int i1, bool stop_after_a, int bb0, int cc0) -> int {
        a.sample0 = b->samples; a.i0 = i0; a.i1 = i1; a.skip_a_first = resume ? 1 : 0; a.stop_after_a = stop_after_a ? 1 : 0;
        a.apply_cfe = resume ? 1 : 0; a.bb_pos = bb0; a.coarse_counter = cc0;
        while (b->next_slice < b->n_slices && b->next_slice * b->slice_len < i1) {   // input slices this segment reads
            JB_CUDA(cudaStreamWaitEvent(b->stream, b->ev_slice[b->next_slice], 0));
            b->next_slice++;
        }
        cudaEvent_t e0 = 0, e1 = 0;
        if (b->profiling) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, b->stream); }
        // OQPSK: the warp-specialised kernel above 8400 bps; 8400 bps (pre-filtered) and lower rates run the single-warp kernel
        int r = (p.kind == JAERO_KIND_MSK) ? msk_pipe_launch(p, a, d_pcm, stride, b->stream)
                : (p.fb > 8400)            ? oqpsk_pipe_launch(p, a, d_pcm, stride, b->stream)
                                           : oqpsk_segment_launch(p, a, d_pcm, stride, b->stream);
        if (b->profiling) { cudaEventRecord(e1, b->stream); b->ev_seg.push_back({e0, e1}); b->prof_samples += (i1 - i0 - (stop_after_a ? 1 : 0)); }
        b->launches++;
        a.new_write = 0;
        return r;
    };
    int bb = b->bb_pos, cc = b->coarse_counter;                   // bb: bbcycbuff_ptr of the reference (= slot in our ring)
    int seg_bb = bb, seg_cc = cc;                                  // counters at the start of the open segment
    for (int i = 0; i < (int)n; i++) {
        // A(i): ring write + trigger test (oqpskdemodulator.cpp:410-429) — lock-step for the whole batch
        bool trigger = false;
        if (cc >= p.Fs || !p.cpu_reduce) {
            bb++; if (bb >= N) bb = 0;
            if (bb % trig_every == 0) trigger = true;
        }
        if (trigger) {
            if (launch(seg_start, i + 1, true, seg_bb, seg_cc)) return JAERO_E_CUDA;
            b->samples += (i - seg_start);                         // samples whose B part has run
            cudaEvent_t c0 = 0, c1 = 0;
            if (b->profiling) { cudaEventCreate(&c0); cudaEventCreate(&c1); cudaEventRecord(c0, b->stream); }
            if (b->cfe.clusters > 0 ? cfe_cluster_run(b->cfe, p, bb, std::min(b->cfe.clusters, p.n_channels), b->stream, &b->launches)
                                    : cfe_run(b->cfe, p, bb, b->stream, &b->launches)) return JAERO_E_CUDA;   // oldest sample at bb
            if (b->profiling) { cudaEventRecord(c1, b->stream); b->ev_cfe.push_back({c0, c1}); }
            b->epochs++;
            // seating check between two launches (the segment kernel has written its ring tiles back; per-channel state is indexed
            // by channel, only the ring rows and chan_of move). A seating that finds no room for its scratch ring sets -1.
            if (b->next_regroup >= 0 && b->epochs >= b->next_regroup) {
                b->next_regroup = b->epochs + (b->epochs < 64 ? 32 : REGROUP_EVERY);
                if (batch_regroup_by_phase(b, false)) return JAERO_E_CUDA;
            }
            cc = 0;                                                // :426
            seg_start = i; resume = true; seg_bb = bb; seg_cc = 0;
        }
        cc++;                                                      // :431
    }
    if (launch(seg_start, (int)n, false, seg_bb, seg_cc)) return JAERO_E_CUDA;
    b->samples += ((int)n - seg_start);
    while (b->next_slice < b->n_slices) { JB_CUDA(cudaStreamWaitEvent(b->stream, b->ev_slice[b->next_slice], 0)); b->next_slice++; }
    b->n_slices = 0; b->next_slice = 0;
    // PeakVolume reads the whole call: only here, after the wait for the last copy slice, is all of it staged (the segments
    // above wait only for the slices they read)
    peak_kernel<<<(p.n_channels + 3) / 4, 128, 0, b->stream>>>(p, d_pcm, stride, (int)n);
    JB_CUDA(cudaGetLastError());
    b->launches++;
    b->bb_pos = bb; b->coarse_counter = cc;
    if (b->pre_on) {                                               // :608 mixer_fir_pre.SetFreq(mixer2_freq_sum/i)
        if (pre_finish_launch(b->pre, p.m2_freq_sum, (int)n, p.Fs, b->stream)) return JAERO_E_CUDA;
        b->launches++;
    }
    return JAERO_OK;
}

int jaero_batch_write(jaero_batch *b, const int16_t *pcm, size_t n, size_t stride)
{
    if (!b || !pcm) { set_error("jaero_batch_write: null argument"); return JAERO_E_ARG; }
    if (n == 0) return JAERO_OK;
    if (stride < n) { set_error("jaero_batch_write: channel_stride < n_samples"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    const size_t C = b->p.n_channels;
    const size_t pitch = (n + 7) & ~(size_t)7;
    if (grow(&b->d_stage, &b->stage_cap, C * pitch, b->stream)) return JAERO_E_CUDA;
    if (n < 8192) {
        JB_CUDA(cudaMemcpy2DAsync(b->d_stage, pitch * sizeof(int16_t), pcm, stride * sizeof(int16_t), n * sizeof(int16_t), C,
                                  cudaMemcpyHostToDevice, b->stream));
        return jaero_batch_write_device(b, b->d_stage, n, pitch);
    }
    // long calls: copy in column slices on a second stream so that the transfer of later samples overlaps the
    // demodulation of earlier ones (pinned host memory makes the copies truly asynchronous)
    if (!b->copy_stream) {
        JB_CUDA(cudaStreamCreateWithFlags(&b->copy_stream, cudaStreamNonBlocking));
        JB_CUDA(cudaEventCreateWithFlags(&b->ev_stage_free, cudaEventDisableTiming));
        for (int k = 0; k < 8; k++) JB_CUDA(cudaEventCreateWithFlags(&b->ev_slice[k], cudaEventDisableTiming));
    }
    JB_CUDA(cudaEventRecord(b->ev_stage_free, b->stream));          // everything already queued that reads the staging buffer
    JB_CUDA(cudaStreamWaitEvent(b->copy_stream, b->ev_stage_free, 0));
    b->slice_len = (int)((((n + 7) / 8) + 7) & ~(size_t)7);
    b->n_slices = 0; b->next_slice = 0;
    for (size_t s0 = 0; s0 < n; s0 += (size_t)b->slice_len) {
        const size_t len = std::min((size_t)b->slice_len, n - s0);
        JB_CUDA(cudaMemcpy2DAsync(b->d_stage + s0, pitch * sizeof(int16_t), pcm + s0, stride * sizeof(int16_t), len * sizeof(int16_t), C,
                                  cudaMemcpyHostToDevice, b->copy_stream));
        JB_CUDA(cudaEventRecord(b->ev_slice[b->n_slices], b->copy_stream));
        b->n_slices++;
    }
    return jaero_batch_write_device(b, b->d_stage, n, pitch);
}

static int pull_ints(jaero_batch *b)
{
    const size_t cp = b->p.cpad;
    JB_CUDA(cudaMemcpyAsync(b->h_ints, b->p.I, (size_t)I_COUNT * cp * sizeof(int), cudaMemcpyDeviceToHost, b->stream));
    JB_CUDA(cudaStreamSynchronize(b->stream));
    return 0;
}

int jaero_batch_read_softbits(jaero_batch *b, int16_t *out, size_t cap, int32_t *counts)
{
    if (!b || !out || !counts) { set_error("jaero_batch_read_softbits: null argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    return drain_softbits(b->p, b->p.I, I_COUNT, I_SOFT_COUNT, I_SOFT_OVERFLOW, b->h_ints, b->h_soft_stage, b->stream, out, cap, counts);
}
int jaero_batch_softbits_device(jaero_batch *b, const int16_t **d_soft, const int32_t **d_counts, size_t *ring_cap)
{
    if (!b || !d_soft || !d_counts || !ring_cap) { set_error("null argument"); return JAERO_E_ARG; }
    *d_soft = b->p.soft; *d_counts = b->p.I + (size_t)I_SOFT_COUNT * b->p.cpad; *ring_cap = (size_t)b->p.soft_cap;
    return JAERO_OK;
}
int jaero_batch_reset_softbits(jaero_batch *b)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    return soft_reset(b->p, b->stream);
}
int jaero_batch_set_dcd(jaero_batch *b, int channel, int dcd)
{
    if (!b || channel >= b->p.n_channels) { set_error("jaero_batch_set_dcd: bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    return launch_set_int(b->p.I + (size_t)I_DCD * b->p.cpad, b->p.n_channels, channel, dcd ? 1 : 0, b->stream);
}
int jaero_batch_set_center_freq(jaero_batch *b, int channel, double hz)
{
    if (!b || channel >= b->p.n_channels) { set_error("jaero_batch_set_center_freq: bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    center_freq_kernel<<<(b->p.n_channels + 127) / 128, 128, 0, b->stream>>>(b->p, channel, hz);
    JB_CUDA(cudaGetLastError());
    return JAERO_OK;
}
// setAFC / setSQL / setCPUReduce (oqpskdemodulator.cpp:149-167, mskdemodulator.cpp:113-131): plain flags the sample loop reads;
// the kernels take them by value at every launch, so a change applies from the next write on
int jaero_batch_set_afc(jaero_batch *b, int state)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->p.afc = state ? 1 : 0;
    return JAERO_OK;
}
int jaero_batch_set_sql(jaero_batch *b, int state)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->p.sql = state ? 1 : 0;
    return JAERO_OK;
}
// connect(demodulator, SignalStatus(bool), aerol, SignalStatusSlot(bool)) (JAERO/mainwindow.cpp:432,508)
int jaero_batch_wire_signal_status(jaero_batch *b, int enabled)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->p.wire_sigstat = enabled ? 1 : 0;
    return JAERO_OK;
}
// Seat the channels of the pipelined 10500 bps kernel: slot_of[c] = seat of channel c (a permutation of 0..n_channels-1), or NULL
// to seat them by symbol-timing phase now. Results never depend on the seating (channels do not interact); throughput does.
int jaero_batch_regroup(jaero_batch *b, const int32_t *slot_of)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    if (!b->d_chan_of) return JAERO_OK;                        // this batch's kernel has a fixed seating
    JB_CUDA(cudaSetDevice(b->device));
    if (!slot_of) return batch_regroup_by_phase(b, true) ? JAERO_E_CUDA : JAERO_OK;
    const int C = b->p.n_channels, cp = b->p.cpad;
    std::vector<int> v(cp), seen(C, 0);
    for (int c = 0; c < C; c++) { if (slot_of[c] < 0 || slot_of[c] >= C || seen[slot_of[c]]) { set_error("jaero_batch_regroup: not a permutation"); return JAERO_E_ARG; } seen[slot_of[c]] = 1; v[c] = slot_of[c]; }
    for (int c = C; c < cp; c++) v[c] = c;
    return batch_apply_seating(b, v) ? JAERO_E_CUDA : JAERO_OK;
}
int jaero_batch_set_cpu_reduce(jaero_batch *b, int state)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->p.cpu_reduce = state ? 1 : 0;
    return JAERO_OK;
}
int jaero_batch_get_status_all(jaero_batch *b, jaero_status *out)
{
    if (!b || !out) { set_error("null argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    const size_t cp = b->p.cpad;
    JB_CUDA(cudaMemcpyAsync(b->h_dbls, b->p.D, (size_t)D_COUNT * cp * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    JB_CUDA(cudaMemcpyAsync(b->h_soft_total, b->p.soft_total, cp * sizeof(long long), cudaMemcpyDeviceToHost, b->stream));
    if (pull_ints(b)) return JAERO_E_CUDA;
    for (int ch = 0; ch < b->p.n_channels; ch++) {
        auto D = [&](int i) { return b->h_dbls[(size_t)i * cp + ch]; };
        auto I = [&](int i) { return b->h_ints[(size_t)i * cp + ch]; };
        jaero_status &s = out[ch];
        s.mixer2_freq = D(D_M2_FREQ); s.mixer2_wtptr = D(D_M2_PTR); s.center_freq = D(D_MC_FREQ);
        s.st_freq = D(D_ST_FREQ); s.st_wtptr = D(D_ST_PTR); s.agc = D(D_AGC_VAL); s.mse = D(D_MSE);
        s.ebno = D(D_EB_EBNO); s.marg = D(D_MARG_VAL); s.cfe_est = D(D_CFE_EST);
        s.n_sig_true = I(I_SIG_TRUE); s.n_sig_false = I(I_SIG_FALSE);
        s.center_wtptr = D(D_MC_PTR); s.st_ref_wtptr = D(D_SR_PTR);
        s.samples = b->samples; s.softbits = b->h_soft_total[ch] + I(I_SOFT_COUNT); s.dcd = I(I_DCD); s.reserved = 0;
        s.peak_volume = (double)I(I_PEAK) / 32768.0;
        s.scatter[0] = D(D_SCAT0_RE); s.scatter[1] = D(D_SCAT0_IM); s.scatter[2] = D(D_SCAT1_RE); s.scatter[3] = D(D_SCAT1_IM);
    }
    // `emit PeakVolume(maxval); maxval=0;`: the read-out restarts the maximum
    JB_CUDA(cudaMemsetAsync(b->p.I + (size_t)I_PEAK * cp, 0, cp * sizeof(int), b->stream));
    return JAERO_OK;
}
int jaero_batch_get_status(jaero_batch *b, int channel, jaero_status *out)
{
    if (!b || !out || channel < 0 || channel >= b->p.n_channels) { set_error("jaero_batch_get_status: bad argument"); return JAERO_E_ARG; }
    std::vector<jaero_status> all(b->p.n_channels);
    int r = jaero_batch_get_status_all(b, all.data());
    if (r) return r;
    *out = all[channel];
    return JAERO_OK;
}

} // extern "C"

// ====================================================================== P- and C-channel frame layers
// The two layers hold the same members; only the parameter block and the per-channel state differ.
template <class Params, class State> struct FrameLayer {
    int device; cudaStream_t stream;
    Params params;
    std::vector<void *> allocs;
    uint8_t *vit_overlap; int *vit_overlap_len, *vit_renorm, *vit_valid;
    int16_t *d_soft_stage; int *d_count_stage; size_t stage_cap;
    State *h_state; uint8_t *h_out;           // pinned: per-channel state; SU records (P) / frame records (C)
    long long launches;
    // Stream ordering between this layer's own stream and a demodulator batch's stream (which the layer never keeps: the
    // batch may be destroyed first). Work launched on a batch's stream is followed by ev_batch, which `stream` waits for;
    // work on `stream` sets own_dirty, and the next call that uses a batch's stream orders that stream behind ev_own.
    cudaEvent_t ev_batch, ev_own; bool own_dirty;
};
struct jaero_pchannel : FrameLayer<PChanParams, PChanState> {};
struct jaero_cchannel : FrameLayer<CChanParams, CChanState> {};

namespace {
// a call is about to launch on a batch's stream `bs`: order it behind whatever this layer queued on its own stream
template <class L> int pc_enter(L *p, cudaStream_t bs)
{
    if (p->own_dirty) { JB_CUDA(cudaEventRecord(p->ev_own, p->stream)); JB_CUDA(cudaStreamWaitEvent(bs, p->ev_own, 0)); p->own_dirty = false; }
    return 0;
}
// ... and the layer's own stream behind what was just launched on `bs` (the batch's stream handle is not kept)
template <class L> int pc_leave(L *p, cudaStream_t bs)
{
    JB_CUDA(cudaEventRecord(p->ev_batch, bs)); JB_CUDA(cudaStreamWaitEvent(p->stream, p->ev_batch, 0));
    return 0;
}
// the frame stage + Viterbi launcher of each layer
int layer_process(jaero_pchannel *p, const int16_t *soft, const int *counts, size_t stride, int *dcd, cudaStream_t s,
                  const int *lost_n = nullptr, const int *lost_pos = nullptr, size_t lost_pitch = 0)
{
    return pchan_process(p->params, soft, counts, (int)stride, dcd, p->vit_overlap, p->vit_overlap_len, p->vit_renorm, p->vit_valid,
                         p->params.queue, s, &p->launches, lost_n, lost_pos, lost_pitch);
}
int layer_process(jaero_cchannel *c, const int16_t *soft, const int *counts, size_t stride, int *dcd, cudaStream_t s,
                  const int *lost_n = nullptr, const int *lost_pos = nullptr, size_t lost_pitch = 0)
{
    return cchan_process(c->params, soft, counts, stride, dcd, c->vit_overlap, c->vit_overlap_len, c->vit_renorm, c->vit_valid,
                         s, &c->launches, lost_n, lost_pos, lost_pitch);
}
template <class L> void layer_destroy(L *l)
{
    if (!l) return;
    cudaSetDevice(l->device);
    cudaDeviceSynchronize();          // work may be queued on a batch's stream, which the layer does not own
    if (l->ev_batch) cudaEventDestroy(l->ev_batch);
    if (l->ev_own) cudaEventDestroy(l->ev_own);
    release(l, {l->d_soft_stage, l->d_count_stage}, {l->h_state, l->h_out}, l->stream);
}
template <class L> int layer_process_batch(L *l, jaero_batch *b, const char *fn)
{
    if (!l || !b || l->params.n_channels != b->p.n_channels || l->device != b->device) { set_error(std::string(fn) + ": batch mismatch"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(l->device));
    const DemodParams &dp = b->p;
    // everything runs on the batch's stream so it is ordered after the demodulator segments
    if (pc_enter(l, b->stream)) return JAERO_E_CUDA;
    if (layer_process(l, dp.soft, dp.I + (size_t)I_SOFT_COUNT * dp.cpad, (size_t)dp.soft_cap, dp.I + (size_t)I_DCD * dp.cpad, b->stream,
                      dp.I + (size_t)I_LOST_N * dp.cpad, dp.lost_pos, dp.cpad)) return JAERO_E_CUDA;
    if (soft_reset(dp, b->stream)) return JAERO_E_CUDA;
    l->launches++;
    return pc_leave(l, b->stream) ? JAERO_E_CUDA : JAERO_OK;
}
// *_process_softbits of the frame layers and the R/T layer: the caller's soft values and counts go to the object's staging pair
template <class O> int stage_softbits(O *o, const int16_t *soft, const int32_t *counts, size_t C, size_t cap)
{
    if (grow(&o->d_soft_stage, &o->stage_cap, C * cap, o->stream, &o->d_count_stage, C)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpyAsync(o->d_soft_stage, soft, C * cap * sizeof(int16_t), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaMemcpyAsync(o->d_count_stage, counts, C * sizeof(int), cudaMemcpyHostToDevice, o->stream));
    return 0;
}
template <class L> int layer_process_softbits(L *l, const int16_t *soft, size_t cap, const int32_t *counts, const char *fn)
{
    if (!l || !soft || !counts || cap == 0) { set_error(std::string(fn) + ": bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(l->device));
    l->own_dirty = true;
    if (stage_softbits(l, soft, counts, l->params.n_channels, cap)) return JAERO_E_CUDA;
    if (layer_process(l, l->d_soft_stage, l->d_count_stage, cap, nullptr, l->stream)) return JAERO_E_CUDA;
    JB_CUDA(cudaStreamSynchronize(l->stream));
    return JAERO_OK;
}
// tick and lost_signal: launch(state, n_channels, args..., demod_dcd, stream), which may write the demodulator's DCD, on the
// batch's stream when a batch is given (b may be NULL: frame layer only). tick passes channel -1.
template <class L, class F, class... A> int layer_dcd_launch(L *l, jaero_batch *b, int channel, const char *fn, F launch, A... args)
{
    if (!l || channel >= l->params.n_channels || (b && b->p.n_channels != l->params.n_channels)) { set_error(std::string(fn) + ": bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(l->device));
    if (b) { if (pc_enter(l, b->stream)) return JAERO_E_CUDA; } else l->own_dirty = true;
    int *dcd = b ? b->p.I + (size_t)I_DCD * b->p.cpad : nullptr;
    if (launch(l->params.state, l->params.n_channels, args..., dcd, b ? b->stream : l->stream)) return JAERO_E_CUDA;
    l->launches++;
    return (b && pc_leave(l, b->stream)) ? JAERO_E_CUDA : JAERO_OK;
}
// Length of the piece of a write that ends in front of the next coarse-estimator trigger sample (the only points where the OQPSK
// demodulator reads DCD and where SignalStatus is emitted): the lock-step counters of jaero_batch_write_device, read-only.
size_t piece_before_next_trigger(const jaero_batch *b, size_t n)
{
    const DemodParams &p = b->p;
    const int N = p.bbnfft, trig_every = p.cpu_reduce ? N : N / 4;
    int bb = b->bb_pos, cc = b->coarse_counter;
    for (size_t i = 0; i < n; i++) {
        if (cc >= p.Fs || !p.cpu_reduce) {
            bb++; if (bb >= N) bb = 0;
            if (bb % trig_every == 0) { if (i > 0) return i; cc = 0; }   // a trigger on the first sample opens this piece
        }
        cc++;
    }
    return n;
}
// writeData with the AeroL attached the way JAERO/mainwindow.cpp:198-237,432,508 wires them: the stream is cut in front of
// every estimator trigger sample and the frame layer runs at each cut, so that the DCD the demodulator reads in
// FreqOffsetEstimateSlot, and the LostSignal that follows a SignalStatus(false), see exactly the soft bits emitted before
// that sample (exact for OQPSK, whose only reads of DCD are in that slot; for MSK the timing-loop gain switches at the next
// cut, at most one estimator epoch after the reference's emit-granular switch). HOST pcm.
template <class L> int layer_write_batch(L *l, jaero_batch *b, const int16_t *pcm, size_t n, size_t stride, const char *fn,
                                         int (*process_batch)(L *, jaero_batch *))
{
    if (!l || !b || !pcm || l->params.n_channels != b->p.n_channels || l->device != b->device) { set_error(std::string(fn) + ": bad argument"); return JAERO_E_ARG; }
    if (stride < n) { set_error(std::string(fn) + ": channel_stride < n_samples"); return JAERO_E_ARG; }
    b->p.wire_sigstat = 1;
    size_t done = 0;
    while (done < n) {
        const size_t k = piece_before_next_trigger(b, n - done);   // >= 1: up to, not including, the next trigger sample
        int rc = jaero_batch_write(b, pcm + done, k, stride);
        if (rc) return rc;
        rc = process_batch(l, b);
        if (rc) return rc;
        done += k;
    }
    return JAERO_OK;
}
template <class L> int pull_state(L *l)
{
    JB_CUDA(cudaMemcpyAsync(l->h_state, l->params.state, (size_t)l->params.n_channels * sizeof(*l->h_state), cudaMemcpyDeviceToHost, l->stream));
    JB_CUDA(cudaStreamSynchronize(l->stream));          // the layer's stream is ordered behind every batch-stream call (pc_leave)
    return 0;
}
template <class L> int layer_get_stats(L *l, int32_t *dcd, int64_t *su_total, int64_t *su_ok)
{
    if (!l) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(l->device));
    if (pull_state(l)) return JAERO_E_CUDA;
    for (int ch = 0; ch < l->params.n_channels; ch++) {
        if (dcd) dcd[ch] = l->h_state[ch].datacd;
        if (su_total) su_total[ch] = l->h_state[ch].su_total;
        if (su_ok) su_ok[ch] = l->h_state[ch].su_ok;
    }
    return JAERO_OK;
}
// Copy-out of a decoded-record queue (R/T packets, C-channel frames): fetch the per-channel state and the queue of `queue`
// records of `rec` bytes per channel, and hand each channel at most `cap` records. A lost record sets *overflow.
template <class State> int read_records(const State *d_state, State *h_state, const uint8_t *d_out, uint8_t *h_out, size_t C, int queue,
                                        size_t rec, cudaStream_t s, uint8_t *out, int cap, int32_t *counts, bool *overflow)
{
    JB_CUDA(cudaMemcpyAsync(h_state, d_state, C * sizeof(State), cudaMemcpyDeviceToHost, s));
    JB_CUDA(cudaMemcpyAsync(h_out, d_out, C * queue * rec, cudaMemcpyDeviceToHost, s));
    JB_CUDA(cudaStreamSynchronize(s));
    for (size_t ch = 0; ch < C; ch++) {
        const int n = h_state[ch].out_count;
        *overflow |= h_state[ch].overflow != 0 || n > cap;
        counts[ch] = n < cap ? n : cap;
        for (int k = 0; k < counts[ch]; k++) memcpy(out + (ch * cap + k) * rec, h_out + (ch * queue + k) * rec, rec);
    }
    return 0;
}
} // namespace

extern "C" {

int jaero_pchannel_create(int n_channels, double fb, int device, jaero_pchannel **out)
{
    if (!out || n_channels <= 0) { set_error("jaero_pchannel_create: bad argument"); return JAERO_E_ARG; }
    const int ifb = (int)(fb + 0.5);
    if (ifb != 600 && ifb != 1200 && ifb != 10500) { set_error("jaero_pchannel_create: P-channel rates are 600, 1200, 10500"); return JAERO_E_ARG; }
    CreateGuard<jaero_pchannel> guard(jaero_pchannel_destroy);
    int r = guard.begin("jaero_pchannel_create", device); if (r) return r;
    jaero_pchannel *p = guard.obj;
    JB_CUDA(cudaEventCreateWithFlags(&p->ev_batch, cudaEventDisableTiming));
    JB_CUDA(cudaEventCreateWithFlags(&p->ev_own, cudaEventDisableTiming));
    PChanParams &pp = p->params;
    pp.n_channels = n_channels; pp.paddinglength = 24;                          // aerol.cpp:940
    switch (ifb) {                                                               // AeroL::setSettings, aerol.cpp:1013-1052
    case 600: pp.cols = 6; pp.number_of_bits = 1152; pp.bits_in_header = 16; pp.total_number_of_bits = 16 + 1152 + 32; pp.oqpsk = 0; pp.dl2_len = 576 - 6 + 1; break;
    case 1200: pp.cols = 9; pp.number_of_bits = 1152; pp.bits_in_header = 16; pp.total_number_of_bits = 16 + 1152 + 32; pp.oqpsk = 0; pp.dl2_len = 576 - 6 + 1; break;
    default: pp.cols = 78; pp.number_of_bits = 4992; pp.bits_in_header = 16 + 178; pp.total_number_of_bits = 16 + 178 + 4992 + 64; pp.oqpsk = 1; pp.dl2_len = 4992 - 6 + 1; break;
    }
    pp.block_len = pp.cols * 64;
    pp.info_cap = pp.number_of_bits / 16 + 16;
    // queue depth: a demodulator soft ring holds max(4096, 2*fb+64) values (jaero_batch_create); a call may hand all of them over
    pp.queue = std::max(PCHAN_QUEUE_MIN, std::max(4096, 2 * ifb + 64) / pp.block_len + 2);
    pp.su_cap = pp.queue * (pp.number_of_bits / 2 / 96) + 8;
    const size_t C = n_channels;
    int rc = 0;
    rc |= owned_alloc(p, &pp.state, C);
    rc |= owned_alloc(p, &pp.blocks, C * pp.queue * pp.block_len);
    rc |= owned_alloc(p, &pp.decoded, C * pp.queue * (pp.block_len / 2));
    rc |= owned_alloc(p, &pp.meta, C * pp.queue);
    rc |= owned_alloc(p, &pp.ready, C);
    rc |= owned_alloc(p, &pp.dl2, C * pp.dl2_len);
    rc |= owned_alloc(p, &pp.infofield, C * pp.info_cap);
    rc |= owned_alloc(p, &pp.su_out, C * pp.su_cap * 16);
    rc |= owned_alloc(p, &p->vit_overlap, C * 64);
    rc |= owned_alloc(p, &p->vit_overlap_len, C);
    rc |= owned_alloc(p, &p->vit_renorm, C);
    rc |= owned_alloc(p, &p->vit_valid, C);
    if (rc) return JAERO_E_CUDA;
    if (frame_set_scrambler() || per_channel_launch(pchan_init_kernel, n_channels, p->stream, pp)) return JAERO_E_CUDA;
    JB_CUDA(cudaStreamSynchronize(p->stream));
    JB_CUDA(cudaMallocHost(&p->h_state, C * sizeof(PChanState)));
    JB_CUDA(cudaMallocHost(&p->h_out, C * pp.su_cap * 16));
    *out = guard.release();
    return JAERO_OK;
}
void jaero_pchannel_destroy(jaero_pchannel *p) { layer_destroy(p); }
int64_t jaero_pchannel_launch_count(const jaero_pchannel *p) { return p ? p->launches : 0; }
int jaero_pchannel_su_capacity(const jaero_pchannel *p) { return p ? p->params.su_cap : 0; }

int jaero_pchannel_process_batch(jaero_pchannel *p, jaero_batch *b) { return layer_process_batch(p, b, "jaero_pchannel_process_batch"); }
int jaero_pchannel_process_softbits(jaero_pchannel *p, const int16_t *soft, size_t cap, const int32_t *counts)
{
    return layer_process_softbits(p, soft, cap, counts, "jaero_pchannel_process_softbits");
}
int jaero_pchannel_tick(jaero_pchannel *p, jaero_batch *b) { return layer_dcd_launch(p, b, -1, "jaero_pchannel_tick", frame_tick<PChanState>); }
// AeroL::SignalStatusSlot(false) -> LostSignal() (aerol.h:920-931): cntr = 1e9, DCD countdown and DCD cleared at once, and
// DataCarrierDetect(false) reaches the demodulator (b may be NULL: frame layer only). channel -1 = every channel.
int jaero_pchannel_lost_signal(jaero_pchannel *p, jaero_batch *b, int channel)
{
    return layer_dcd_launch(p, b, channel, "jaero_pchannel_lost_signal", frame_lost<PChanState>, channel);
}
int jaero_pchannel_write_batch(jaero_pchannel *p, jaero_batch *b, const int16_t *pcm, size_t n, size_t stride)
{
    return layer_write_batch(p, b, pcm, n, stride, "jaero_pchannel_write_batch", jaero_pchannel_process_batch);
}
int jaero_pchannel_read_sus(jaero_pchannel *p, uint8_t *out, size_t cap, int32_t *counts)
{
    if (!p || !out || !counts) { set_error("jaero_pchannel_read_sus: null argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(p->device));
    if (pull_state(p)) return JAERO_E_CUDA;
    const PChanParams &pp = p->params;
    bool overflow = false; int maxc = 0;
    for (int ch = 0; ch < pp.n_channels; ch++) { maxc = std::max(maxc, p->h_state[ch].su_count); overflow |= p->h_state[ch].queue_overflow != 0 || (size_t)p->h_state[ch].su_count > cap; }
    if (overflow) { set_error("P-channel queue overflow: call process/read more often"); return JAERO_E_OVERFLOW; }
    if (maxc) { JB_CUDA(cudaMemcpyAsync(p->h_out, pp.su_out, (size_t)pp.n_channels * pp.su_cap * 16, cudaMemcpyDeviceToHost, p->stream)); JB_CUDA(cudaStreamSynchronize(p->stream)); }
    for (int ch = 0; ch < pp.n_channels; ch++) {
        counts[ch] = p->h_state[ch].su_count;
        if (counts[ch]) memcpy(out + (size_t)ch * cap * 16, p->h_out + (size_t)ch * pp.su_cap * 16, (size_t)counts[ch] * 16);
    }
    if (per_channel_launch(pchan_su_reset_kernel, pp.n_channels, p->stream, pp)) return JAERO_E_CUDA;
    p->own_dirty = true;
    return JAERO_OK;
}
int jaero_pchannel_discard_sus(jaero_pchannel *p)
{
    if (!p) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(p->device));
    if (per_channel_launch(pchan_su_reset_kernel, p->params.n_channels, p->stream, p->params)) return JAERO_E_CUDA;
    p->own_dirty = true;
    p->launches++;
    return JAERO_OK;
}
int jaero_pchannel_get_stats(jaero_pchannel *p, int32_t *dcd, int64_t *su_total, int64_t *su_ok) { return layer_get_stats(p, dcd, su_total, su_ok); }

} // extern "C"

// ====================================================================== burst MSK demodulator
struct jaero_burst {
    int device; cudaStream_t stream;
    BurstParams p; FastFir hil;
    std::vector<void *> allocs;
    long long samples;
    int16_t *d_stage; size_t stage_cap;
    double2 *tw32k, *wa, *wb; int *d_ev_list; int ev_round;
    int *h_ints; double *h_dbls; int16_t *h_soft;
    std::vector<int> h_ev;
    long long launches;
};

namespace {
__global__ void burst_init_kernel(BurstParams p, double freq_center, double st_freq)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= p.cpad) return;
    auto D = [&](int i) -> double & { return p.BD[(size_t)i * p.cpad + ch]; };
    auto I = [&](int i) -> int & { return p.BI[(size_t)i * p.cpad + ch]; };
    const double sr = (double)((float)((int)p.Fs));
    D(BD_M2_FREQ) = freq_center; D(BD_M2_STEP) = (freq_center) * ((double)jb::WTSIZE) / sr;
    D(BD_MC_FREQ) = freq_center; D(BD_MC_STEP) = (freq_center) * ((double)jb::WTSIZE) / sr;
    D(BD_ST_FREQ) = st_freq; D(BD_ST_STEP) = (st_freq) * ((double)jb::WTSIZE) / sr;
    D(BD_SH_FREQ) = st_freq; D(BD_SH_STEP) = (st_freq) * ((double)jb::WTSIZE) / sr;
    D(BD_MSE) = 10.0;                                    // burstmskdemodulator.cpp:195
    D(BD_ROT_RE) = 1.0; D(BD_SAV_RE) = 1.0;              // rotator=1, symboltone_averotator=1 (:201-202); symboltone_rotator stays 0
    D(BD_DIFF_LAST) = -1.0;
    if (p.kind == 1) {                                   // burst OQPSK ctor (burstoqpskdemodulator.cpp:4-133)
        D(BD_MSE) = 100.0; D(BD_VOL_GAIN) = 1.0; D(BD_STR_RE) = 1.0;     // symboltone_rotator=1, never reset
        D(BD_ST_FREQ) = 10500.0; D(BD_ST_STEP) = (10500.0) * ((double)jb::WTSIZE) / sr;
        D(BD_SR_FREQ) = 10500.0; D(BD_SR_STEP) = (10500.0) * ((double)jb::WTSIZE) / sr;
        D(BD_SH_FREQ) = 10500.0 / 4.0; D(BD_SH_STEP) = (10500.0 / 4.0) * ((double)jb::WTSIZE) / sr;
    }
    I(BI_PD_CNTDOWN) = 2 * p.pd_len; I(BI_PD_MAXPOSCNT) = -1;    // PeakDetector::setSettings (DSP.h:502-513)
    I(BI_STARTSTOP) = -1;                                // ctor :69
}
} // namespace

extern "C" {

static int burst_create(const jaero_settings *s, int n_channels, int device, int kind, jaero_burst **out)
{
    if (!s || !out || n_channels <= 0) { set_error("jaero_burst_create: bad argument"); return JAERO_E_ARG; }
    if (kind == 0 && (s->Fs != 48000 || (s->fb != 600 && s->fb != 1200))) { set_error("jaero_burst_msk_create: burst MSK runs at Fs=48000 with fb 600 or 1200"); return JAERO_E_ARG; }
    if (kind == 1 && (s->Fs != 48000 || s->fb != 10500)) { set_error("jaero_burst_oqpsk_create: burst OQPSK runs at Fs=48000, fb=10500"); return JAERO_E_ARG; }
    CreateGuard<jaero_burst> guard(jaero_burst_destroy);
    { int r = guard.begin("jaero_burst_msk_create", device); if (r) return r; }
    jaero_burst *b = guard.obj;
    BurstParams &p = b->p;
    p.kind = kind; p.sql = s->sql;
    p.n_channels = n_channels; p.cpad = (n_channels + 31) & ~31;
    p.Fs = s->Fs; p.fb = s->fb; p.lockingbw = s->lockingbw; p.signalthreshold = s->signalthreshold; p.afc = 1;   // ctor: afc=true (:15)
    double fc = s->freq_center;
    if (fc > ((p.Fs / 2.0) - (p.lockingbw / 2.0))) fc = ((p.Fs / 2.0) - (p.lockingbw / 2.0));
    p.sps = (int)(p.Fs / p.fb);
    const double SPS = kind == 1 ? 2.0 * p.Fs / p.fb : (double)p.sps;            // burstoqpskdemodulator.cpp:219
    p.spsd = SPS;
    std::vector<double> taps;
    if (kind == 1) { p.sps = (int)SPS; p.ntaps = 55; taps = rrc_taps(1.0, 55, 48000, 10500 / 2.0); }    // ctor :38-46
    else {
        p.ntaps = 2 * p.sps;
        if (p.ntaps > MAX_TAPS) { set_error("burst MSK: matched filter too long"); return JAERO_E_ARG; }
        taps.resize(p.ntaps);
        for (int i = 0; i < p.ntaps; i++) taps[i] = sin(M_PI * i / (2.0 * SPS)) / (2.0 * SPS);      // :173-177
    }
    for (int k = 0; k < p.ntaps; k++) p.taps[k] = taps[k];
    p.agc_len = (int)round(1 * p.Fs);
    auto qround = [](double d) { return d >= 0.0 ? int(d + 0.5) : int(d - double(int(d - 1)) + 0.5) + int(d - 1); };
    double btdiff_fd = 0;
    if (kind == 1) {                                              // burstoqpskdemodulator.cpp:202-277
        p.btma_len = qround(128.0 * SPS); p.mav1_len = (int)(SPS * 128); btdiff_fd = SPS * 128; p.btdiff_len = (int)std::ceil(btdiff_fd) + 1;
        p.pd_len = (int)(SPS * 128.0 / 2.0); p.pd_threshold = 0.2;
        p.tri_sz = qround((256.0 + 16.0 + 16.0) * SPS); p.d1_len = (int)(SPS * 128.0 * 2.5 - 190) + 1; p.d2_len = p.tri_sz + 1;
        p.tri_nb = p.tri_nt = qround(128.0 * SPS);
        p.res_b0 = 0.0048847995518126464; p.res_b1 = 0; p.res_b2 = -0.0048847995518126464;       // ctor :69-75 (75 Hz)
        p.res_a1 = -0.3882746897971619; p.res_a2 = 0.99023040089637471;
        p.ee = 0.4;
    } else if (p.fb >= 1200) {                                           // :205-256
        p.btma_len = qround(126.0 * SPS); p.mav1_len = (int)(SPS * 126); p.btdiff_len = (int)std::ceil(SPS * 126) + 1;
        p.pd_len = (int)(SPS * 126.0 / 2.0); p.pd_threshold = 0.1;
        p.tri_sz = qround(200.0 * SPS); p.d1_len = ((int)289 * p.sps) + 20 + 1; p.d2_len = (int)(qround(72 + 120.0) * SPS) + 1;
        p.size_base = 126; p.size_top = 74; p.start_processing = 120; p.end_rotation = (int)((120 + 37) * SPS);
        p.res_a1 = -1.993312819378528; p.res_a2 = 0.999476538254407; p.res_b0 = 2.617308727964618e-04; p.res_b1 = 0; p.res_b2 = -2.617308727964618e-04;
        p.ee = 0.025; btdiff_fd = SPS * 126;
    } else {                                                      // :257-311
        p.btma_len = qround(150.0 * SPS); p.mav1_len = (int)(SPS * 150); p.btdiff_len = (int)std::ceil(SPS * 150) + 1;
        p.pd_len = (int)(SPS * 150.0 / 2.0); p.pd_threshold = 0.2;
        p.tri_sz = qround(224 * SPS); p.d1_len = ((int)397 * p.sps) + 20 + 1; p.d2_len = qround((72 + 150.0) * SPS) + 1;
        p.size_base = 150; p.size_top = 74; p.start_processing = 150; p.end_rotation = (int)((150 + 56) * SPS);
        p.res_a1 = -1.991228154418550; p.res_a2 = 0.997385427096603; p.res_b0 = 0.001307286451699; p.res_b1 = 0; p.res_b2 = -0.001307286451699;
        p.ee = 0.015; btdiff_fd = SPS * 150;
    }
    if (kind == 0) { p.tri_nb = (int)rint(p.size_base * SPS); p.tri_nt = (int)rint(p.size_top * SPS); }
    if ((BURST_CHUNK - 1) / (p.tri_sz + 1) + 2 > BURST_MAXEV) { set_error("burst: more trident fills per chunk than buffer slots"); return JAERO_E_ARG; }
    p.startstopstart = kind == 1 ? (int)(SPS * (1050)) : (int)(SPS * 500);
    p.btd1_len = (int)std::ceil(1.0 * SPS) + 1;
    int kk;
    std::vector<double> w_btd1, w_btdiff, w_a1, w_tmp;
    if (!delay_table(1.0 * SPS, INT_MAX, w_btd1, &kk) || !delay_table(btdiff_fd, INT_MAX, w_btdiff, &kk) || !delay_table(SPS / 2.0, INT_MAX, w_a1, &p.a1_k)) {
        set_error("burst: unsupported delay"); return JAERO_E_ARG; }
    if (kind == 0) {
        msk_half_symbol_delay(p.sps, p.d8_k, p.d8_w);           // d8: Delay<double>(SPS/2)
        p.eb_len = (int)(0.15 * p.Fs); p.agc2_len = (int)round((SPS * 128.0 / p.Fs) * p.Fs); p.ds_len = p.sps + 1; p.msema_len = 75;
    } else {
        const double sps0 = 2.0 * 48000 / 10500;                  // ctor :48-52
        if (!delay_table4(sps0 / 4.0, p.w41v, &p.k41) || !delay_table4(sps0 / 8.0, p.w8v, &p.k8)) { set_error("burst OQPSK: unsupported delay"); return JAERO_E_ARG; }
        p.d8_k = 1; p.ds_len = 1;
        p.eb_len = (int)(SPS * (256.0)); p.agc2_len = (int)round((SPS * 64.0 / p.Fs) * p.Fs); p.msema_len = 128;
    }
    p.soft_cap = std::max(4096, (int)(2 * p.fb) + 64);
    const size_t cp = p.cpad, C = n_channels;
    int rc = 0;
    rc |= owned_alloc(b, &p.BD, (size_t)BD_COUNT * cp); rc |= owned_alloc(b, &p.BI, (size_t)BI_COUNT * cp);
    rc |= owned_alloc(b, &p.agc_ring, (size_t)p.agc_len * cp); rc |= owned_alloc(b, &p.d1_ring, (size_t)p.d1_len * cp);
    rc |= owned_alloc(b, &p.d2_ring, (size_t)p.d2_len * cp); rc |= owned_alloc(b, &p.btd1_ring, (size_t)p.btd1_len * cp);
    rc |= owned_alloc(b, &p.btma_ring, (size_t)p.btma_len * cp); rc |= owned_alloc(b, &p.mav1_ring, (size_t)p.mav1_len * cp);
    rc |= owned_alloc(b, &p.btdiff_ring, (size_t)p.btdiff_len * cp);
    rc |= owned_alloc(b, &p.pd1_ring, (size_t)(2 * p.pd_len + 1) * cp); rc |= owned_alloc(b, &p.pd2_ring, (size_t)(p.pd_len + 1) * cp);
    rc |= owned_alloc(b, &p.pd3_ring, (size_t)(2 * p.pd_len + 1) * cp);
    rc |= owned_alloc(b, &p.a1_ring, (size_t)(p.a1_k + 1) * cp); rc |= owned_alloc(b, &p.eb1_ring, (size_t)p.eb_len * cp);
    rc |= owned_alloc(b, &p.eb2_ring, (size_t)p.eb_len * cp); rc |= owned_alloc(b, &p.agc2_ring, (size_t)p.agc2_len * cp);
    rc |= owned_alloc(b, &p.d8_ring, (size_t)(p.d8_k + 1) * cp); rc |= owned_alloc(b, &p.msema_ring, (size_t)p.msema_len * cp);
    rc |= owned_alloc(b, &p.fir_re, (size_t)(p.ntaps + 1) * cp); rc |= owned_alloc(b, &p.fir_im, (size_t)(p.ntaps + 1) * cp);
    rc |= owned_alloc(b, &p.ds_ring, (size_t)p.ds_len * cp);
    rc |= owned_alloc(b, &p.tri, C * BURST_MAXEV * p.tri_sz); rc |= owned_alloc(b, &p.ev_sample, C * BURST_MAXEV);
    rc |= owned_alloc(b, &p.ev_result, C * BURST_MAXEV * 8);
    p.astride = BURST_CHUNK;
    rc |= owned_alloc(b, &p.analytic, C * p.astride); rc |= owned_alloc(b, &p.vtd, C * p.astride);
    rc |= owned_alloc(b, &p.soft, C * p.soft_cap);
    {
        double *d1 = 0, *d2 = 0, *d3 = 0;
        rc |= owned_alloc(b, &d1, w_btd1.size()); rc |= owned_alloc(b, &d2, w_btdiff.size()); rc |= owned_alloc(b, &d3, w_a1.size());
        if (!rc) {
            JB_CUDA(cudaMemcpyAsync(d1, w_btd1.data(), w_btd1.size() * 8, cudaMemcpyHostToDevice, b->stream));
            JB_CUDA(cudaMemcpyAsync(d2, w_btdiff.data(), w_btdiff.size() * 8, cudaMemcpyHostToDevice, b->stream));
            JB_CUDA(cudaMemcpyAsync(d3, w_a1.data(), w_a1.size() * 8, cudaMemcpyHostToDevice, b->stream));
            JB_CUDA(cudaStreamSynchronize(b->stream));
        }
        p.btd1_wv = d1; p.btdiff_wv = d2; p.a1_wv = d3;
    }
    b->ev_round = 128;
    rc |= owned_alloc(b, &b->tw32k, (size_t)TRI_N); rc |= owned_alloc(b, &b->wa, (size_t)2 * b->ev_round * TRI_N); rc |= owned_alloc(b, &b->wb, (size_t)2 * b->ev_round * TRI_N);
    rc |= owned_alloc(b, &b->d_ev_list, (size_t)2 * C * BURST_MAXEV);
    if (rc) return JAERO_E_CUDA;
    {   // Hilbert filter: QJHilbertFilter::setSize(2048) (DSP.cpp:759-789), streaming FFT convolution nfft 8192
        const int N = 2048;
        std::vector<std::complex<double>> hk(N);
        for (int i = 0; i < N; i++) {
            if (i == N / 2) hk[i] = std::complex<double>(-1, 0);
            else if ((i % 2) == 0) hk[i] = 0;
            else hk[i] = std::complex<double>(0, (2.0 / ((double)N)) / (std::tan(M_PI * (((double)i) / ((double)N) - 0.5))));
        }
        int r = fastfir_create(b, hk, 8192, n_channels, b->hil);
        if (r) return r;
    }
    {
        std::vector<double> wt;
        if (upload_wave_table(b, wt, &p.sin_t, &p.cos_t)) return JAERO_E_CUDA;
        const std::vector<std::complex<double>> tw32 = twiddles(TRI_N);
        JB_CUDA(cudaMemcpyAsync(b->tw32k, tw32.data(), (size_t)TRI_N * 16, cudaMemcpyHostToDevice, b->stream));
        JB_CUDA(cudaStreamSynchronize(b->stream));
    }
    burst_init_kernel<<<(p.cpad + 127) / 128, 128, 0, b->stream>>>(p, fc, p.fb / 2.0);
    JB_CUDA(cudaGetLastError());
    JB_CUDA(cudaStreamSynchronize(b->stream));
    JB_CUDA(cudaMallocHost(&b->h_ints, (size_t)BI_COUNT * cp * sizeof(int)));
    JB_CUDA(cudaMallocHost(&b->h_dbls, (size_t)BD_COUNT * cp * sizeof(double)));
    JB_CUDA(cudaMallocHost(&b->h_soft, C * p.soft_cap * sizeof(int16_t)));
    *out = guard.release();
    return JAERO_OK;
}
int jaero_burst_msk_create(const jaero_settings *s, int n_channels, int device, jaero_burst **out) { return burst_create(s, n_channels, device, 0, out); }
int jaero_burst_oqpsk_create(const jaero_settings *s, int n_channels, int device, jaero_burst **out) { return burst_create(s, n_channels, device, 1, out); }
void jaero_burst_destroy(jaero_burst *b)
{
    if (!b) return;
    cudaSetDevice(b->device);
    cudaStreamSynchronize(b->stream);
    release(b, {b->d_stage}, {b->h_ints, b->h_dbls, b->h_soft}, b->stream);
}
int64_t jaero_burst_launch_count(const jaero_burst *b) { return b ? b->launches : 0; }
int jaero_burst_sync(jaero_burst *b) { return sync_stream(b); }
int jaero_burst_write_device(jaero_burst *b, const int16_t *d_pcm, size_t n, size_t stride)
{
    if (!b || !d_pcm) { set_error("jaero_burst_write_device: null argument"); return JAERO_E_ARG; }
    if (n == 0) return JAERO_OK;
    if (stride < n || n > 0x7fffffff) { set_error("jaero_burst_write_device: bad stride / length"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    const BurstParams &p = b->p;
    const size_t cp = p.cpad;
    int new_write = 1;
    for (size_t c0 = 0; c0 < n; c0 += BURST_CHUNK) {
        const int m = (int)std::min((size_t)BURST_CHUNK, n - c0);
        // Hilbert transform of this chunk (JFastFir::update: per-sample exchange + block transforms)
        if (fastfir_feed(b->hil, m, p.n_channels, b->stream, &b->launches, [&](int i0, int i1, int fill0) {
                return hilbert_exchange_launch(b->hil, p, d_pcm, stride, (int)c0, i0, i1, fill0, b->stream); }))
            return JAERO_E_CUDA;
        if (burst_front_launch(p, b->samples, m, b->stream)) return JAERO_E_CUDA;
        b->launches++;
        // trident events of this chunk
        JB_CUDA(cudaMemcpyAsync(b->h_ints, p.BI + (size_t)BI_NEV * cp, cp * sizeof(int), cudaMemcpyDeviceToHost, b->stream));
        JB_CUDA(cudaStreamSynchronize(b->stream));
        b->h_ev.clear();
        for (int ch = 0; ch < p.n_channels; ch++) for (int e = 0; e < b->h_ints[ch]; e++) { b->h_ev.push_back(ch); b->h_ev.push_back(e); }
        const int nevt = (int)b->h_ev.size() / 2;
        if (nevt) JB_CUDA(cudaMemcpyAsync(b->d_ev_list, b->h_ev.data(), b->h_ev.size() * sizeof(int), cudaMemcpyHostToDevice, b->stream));
        for (int e0 = 0; e0 < nevt; e0 += b->ev_round) {
            const int cnt = std::min(b->ev_round, nevt - e0);
            if (burst_trident_fft_launch(p, b->d_ev_list + 2 * e0, cnt, b->wa, b->wb, b->tw32k, b->stream)) return JAERO_E_CUDA;
            b->launches += 2;
        }
        if (burst_back_launch(p, b->samples, m, new_write, b->stream)) return JAERO_E_CUDA;
        new_write = 0;
        b->launches++;
        b->samples += m;
    }
    return JAERO_OK;
}
int jaero_burst_write(jaero_burst *b, const int16_t *pcm, size_t n, size_t stride)
{
    if (!b || !pcm) { set_error("jaero_burst_write: null argument"); return JAERO_E_ARG; }
    if (n == 0) return JAERO_OK;
    if (stride < n) { set_error("jaero_burst_write: channel_stride < n_samples"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    const size_t C = b->p.n_channels, pitch = (n + 7) & ~(size_t)7;
    if (grow(&b->d_stage, &b->stage_cap, C * pitch, b->stream)) return JAERO_E_CUDA;
    JB_CUDA(cudaMemcpy2DAsync(b->d_stage, pitch * 2, pcm, stride * 2, n * 2, C, cudaMemcpyHostToDevice, b->stream));
    return jaero_burst_write_device(b, b->d_stage, n, pitch);
}
int jaero_burst_read_softbits(jaero_burst *b, int16_t *out, size_t cap, int32_t *counts)
{
    if (!b || !out || !counts) { set_error("jaero_burst_read_softbits: null argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    return drain_softbits(b->p, b->p.BI, BI_COUNT, BI_SOFT_COUNT, BI_SOFT_OVERFLOW, b->h_ints, b->h_soft, b->stream, out, cap, counts);
}
int jaero_burst_set_dcd(jaero_burst *b, int channel, int dcd)
{
    if (!b || channel >= b->p.n_channels) { set_error("jaero_burst_set_dcd: bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    return launch_set_int(b->p.BI + (size_t)BI_DCD * b->p.cpad, b->p.n_channels, channel, dcd ? 1 : 0, b->stream);
}
int jaero_burst_set_afc(jaero_burst *b, int state)                  // burstmskdemodulator.cpp / burstoqpskdemodulator.cpp setAFC
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->p.afc = state ? 1 : 0;
    return JAERO_OK;
}
int jaero_burst_set_sql(jaero_burst *b, int state)
{
    if (!b) { set_error("null handle"); return JAERO_E_ARG; }
    b->p.sql = state ? 1 : 0;
    return JAERO_OK;
}
int jaero_burst_get_status_all(jaero_burst *b, jaero_burst_status *out)
{
    if (!b || !out) { set_error("null argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(b->device));
    const size_t cp = b->p.cpad;
    JB_CUDA(cudaMemcpyAsync(b->h_dbls, b->p.BD, (size_t)BD_COUNT * cp * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
    JB_CUDA(cudaMemcpyAsync(b->h_ints, b->p.BI, (size_t)BI_COUNT * cp * sizeof(int), cudaMemcpyDeviceToHost, b->stream));
    JB_CUDA(cudaStreamSynchronize(b->stream));
    for (int ch = 0; ch < b->p.n_channels; ch++) {
        auto D = [&](int i) { return b->h_dbls[(size_t)i * cp + ch]; };
        auto I = [&](int i) { return b->h_ints[(size_t)i * cp + ch]; };
        jaero_burst_status &s = out[ch];
        s.mixer2_freq = D(BD_M2_FREQ); s.mixer2_wtptr = D(BD_M2_PTR); s.center_freq = D(BD_MC_FREQ); s.st_freq = D(BD_ST_FREQ); s.st_wtptr = D(BD_ST_PTR);
        s.agc = D(BD_AGC_VAL); s.mse = D(BD_MSE); s.ebno = D(BD_EB_EBNO); s.vol_gain = D(BD_VOL_GAIN); s.rotator_freq = D(BD_ROT_FREQ);
        s.n_sig_true = I(BI_SIG_TRUE); s.n_sig_false = I(BI_SIG_FALSE); s.cntr = I(BI_CNTR); s.startstop = I(BI_STARTSTOP);
        s.last_burst_ebno = D(BD_LAST_EBNO_EMIT); s.n_ebno_emits = I(BI_EBNO_EMITS);
    }
    return JAERO_OK;
}

// ---- test support: the trident FFTs and peak searches on caller segments (not part of the drop-in surface)
int jaero_burst_trident_geometry(const jaero_burst *b, int32_t out[4])
{
    if (!b || !out) { set_error("jaero_burst_trident_geometry: null argument"); return JAERO_E_ARG; }
    out[0] = b->p.tri_sz; out[1] = b->p.tri_nb; out[2] = b->p.tri_nt; out[3] = TRI_N;
    return JAERO_OK;
}
int jaero_burst_probe_trident(jaero_burst *b, int n_events, const int32_t *ev_channel, const int32_t *ev_slot, const double *segments,
                              const double *spectra_in, double *spectra_out, double *result)
{
    if (!b || n_events <= 0 || !ev_channel || !ev_slot || (!segments && !spectra_in) || !result) {
        set_error("jaero_burst_probe_trident: null argument or n_events <= 0"); return JAERO_E_ARG; }
    BurstParams &p = b->p;
    const int C = p.n_channels;
    // event e of the probe is event number ev[e] of its channel, in the order given, and its fill sits in slot ev_slot[e]:
    // the kernels find the slot through ev_sample's slot field, as after burst_front
    std::vector<int> ev_count(C, 0), ev_list(2 * (size_t)n_events), ev_table((size_t)C * BURST_MAXEV, 0);
    std::vector<char> used((size_t)C * BURST_MAXEV, 0);
    for (int e = 0; e < n_events; e++) {
        const int ch = ev_channel[e], slot = ev_slot[e];
        if (ch < 0 || ch >= C) { set_error("jaero_burst_probe_trident: event " + std::to_string(e) + ": channel out of range"); return JAERO_E_ARG; }
        if (slot < 0 || slot >= BURST_MAXEV) { set_error("jaero_burst_probe_trident: event " + std::to_string(e) + ": slot outside [0, BURST_MAXEV)"); return JAERO_E_ARG; }
        if (used[(size_t)ch * BURST_MAXEV + slot]) { set_error("jaero_burst_probe_trident: event " + std::to_string(e) + ": (channel, slot) appears twice"); return JAERO_E_ARG; }
        used[(size_t)ch * BURST_MAXEV + slot] = 1;
        const int ev = ev_count[ch]++;
        ev_list[2 * e] = ch; ev_list[2 * e + 1] = ev;
        ev_table[(size_t)ch * BURST_MAXEV + ev] = ev | (slot << 24);
    }
    JB_CUDA(cudaSetDevice(b->device));
    const cudaStream_t s = b->stream;
    JB_CUDA(cudaStreamSynchronize(s));
    // every copy below reads host memory that stays alive until the final synchronisation
    if (!spectra_in)
        for (int e = 0; e < n_events; e++)
            JB_CUDA(cudaMemcpyAsync(p.tri + ((size_t)ev_channel[e] * BURST_MAXEV + ev_slot[e]) * p.tri_sz, segments + (size_t)e * p.tri_sz,
                                    (size_t)p.tri_sz * sizeof(double), cudaMemcpyHostToDevice, s));
    JB_CUDA(cudaMemcpyAsync(p.ev_sample, ev_table.data(), ev_table.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    JB_CUDA(cudaMemcpyAsync(b->d_ev_list, ev_list.data(), ev_list.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    const size_t spec = (size_t)2 * TRI_N * 2;                         // doubles per event: base then top, complex
    for (int e0 = 0; e0 < n_events; e0 += b->ev_round) {               // rounds as jaero_burst_write_device runs them
        const int cnt = std::min(b->ev_round, n_events - e0);
        if (spectra_in) {
            JB_CUDA(cudaMemcpyAsync(b->wb, spectra_in + e0 * spec, cnt * spec * sizeof(double), cudaMemcpyHostToDevice, s));
            if (burst_trident_peaks_launch(p, b->d_ev_list + 2 * e0, cnt, b->wa, b->wb, s)) return JAERO_E_CUDA;
        } else if (burst_trident_fft_launch(p, b->d_ev_list + 2 * e0, cnt, b->wa, b->wb, b->tw32k, s)) return JAERO_E_CUDA;
        if (spectra_out) JB_CUDA(cudaMemcpyAsync(spectra_out + e0 * spec, b->wb, cnt * spec * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    std::vector<double> res((size_t)C * BURST_MAXEV * 8);
    JB_CUDA(cudaMemcpyAsync(res.data(), p.ev_result, res.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    JB_CUDA(cudaStreamSynchronize(s));
    for (int e = 0; e < n_events; e++)
        for (int q = 0; q < 5; q++) result[5 * e + q] = res[((size_t)ev_list[2 * e] * BURST_MAXEV + ev_list[2 * e + 1]) * 8 + q];
    return JAERO_OK;
}

} // extern "C"

// ====================================================================== R/T burst channel layer (§8(f)2)

struct jaero_rt {
    int device; cudaStream_t stream;
    RtParams rp;
    std::vector<void *> allocs;
    int16_t *d_soft_stage; int *d_count_stage; size_t stage_cap;
    RtState *h_state; uint8_t *h_out;
    long long launches;
    int vector_mode;
};

extern "C" {

int jaero_rt_create(double fb, int n_channels, int device, jaero_rt **out)
{
    if (!out || n_channels <= 0) { set_error("jaero_rt_create: bad argument"); return JAERO_E_ARG; }
    const int ifb = (int)(fb >= 0.0 ? fb + 0.5 : fb - 0.5);
    if (ifb != 600 && ifb != 1200 && ifb != 10500) { set_error("jaero_rt_create: burst R/T channels run at 600, 1200 or 10500 bps"); return JAERO_E_ARG; }
    CreateGuard<jaero_rt> guard(jaero_rt_destroy);
    { int e = guard.begin("jaero_rt_create", device); if (e) return e; }
    jaero_rt *r = guard.obj;
    RtParams &rp = r->rp;
    rp.n_channels = n_channels; rp.ifb = ifb; rp.oqpsk = (ifb == 10500);
    rp.number_of_bits = (ifb == 10500) ? 4992 : 1152;                       // aerol.cpp:1012-1050
    rp.total_number_of_bits = rp.oqpsk ? ifb : ifb * 3;                     // :1062-1070
    const size_t C = n_channels;
    int rc = 0;
    rc |= owned_alloc(r, &rp.state, C); rc |= owned_alloc(r, &rp.slots, C * RT_SLOTS); rc |= owned_alloc(r, &rp.blocks, C * RT_SLOTS * RT_BLOCK);
    rc |= owned_alloc(r, &rp.out, C * RT_OUT * RT_OUT_BYTES);
    if (rc) return JAERO_E_CUDA;
    if (frame_set_scrambler() || per_channel_launch(rt_init_kernel, n_channels, r->stream, rp)) return JAERO_E_CUDA;
    JB_CUDA(cudaStreamSynchronize(r->stream));
    JB_CUDA(cudaMallocHost(&r->h_state, C * sizeof(RtState)));
    JB_CUDA(cudaMallocHost(&r->h_out, C * RT_OUT * RT_OUT_BYTES));
    *out = guard.release();
    return JAERO_OK;
}
void jaero_rt_destroy(jaero_rt *r)
{
    if (!r) return;
    cudaSetDevice(r->device);
    cudaStreamSynchronize(r->stream);
    release(r, {r->d_soft_stage, r->d_count_stage}, {r->h_state, r->h_out}, r->stream);
}
int64_t jaero_rt_launch_count(const jaero_rt *r) { return r ? r->launches : 0; }

int jaero_rt_process_softbits(jaero_rt *r, const int16_t *soft, size_t cap, const int32_t *counts)
{
    if (!r || !soft || !counts || cap == 0) { set_error("jaero_rt_process_softbits: bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(r->device));
    if (stage_softbits(r, soft, counts, r->rp.n_channels, cap)) return JAERO_E_CUDA;
    if (rt_process(r->rp, r->d_soft_stage, r->d_count_stage, cap, r->stream, &r->launches, r->vector_mode ? -1 : 0)) return JAERO_E_CUDA;
    JB_CUDA(cudaStreamSynchronize(r->stream));
    return JAERO_OK;
}
int jaero_rt_process_burst(jaero_rt *r, jaero_burst *b)
{
    if (!r || !b || r->rp.n_channels != b->p.n_channels || r->device != b->device) { set_error("jaero_rt_process_burst: demodulator mismatch"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(r->device));
    const BurstParams &bp = b->p;
    JB_CUDA(cudaStreamSynchronize(r->stream));
    // on the demodulator's stream: ordered after its kernels; its soft ring is drained afterwards
    if (rt_process(r->rp, bp.soft, bp.BI + (size_t)BI_SOFT_COUNT * bp.cpad, (size_t)bp.soft_cap, b->stream, &r->launches,
                   r->vector_mode ? (bp.kind == 1 ? 32 : 12) : 0)) return JAERO_E_CUDA;   // emit sizes: burstoqpskdemodulator.cpp / burstmskdemodulator.cpp:735
    if (soft_reset(bp, b->stream)) return JAERO_E_CUDA;
    r->launches++;
    JB_CUDA(cudaStreamSynchronize(b->stream));
    return JAERO_OK;
}
// Opt-in: reproduce AeroL::Decode's return in the middle of a soft-bit vector when the burst time-out fires (aerol.cpp:2018-2027)
int jaero_rt_set_vector_mode(jaero_rt *r, int enabled)
{
    if (!r) { set_error("null handle"); return JAERO_E_ARG; }
    r->vector_mode = enabled ? 1 : 0;
    return JAERO_OK;
}
int jaero_rt_tick(jaero_rt *r)
{
    if (!r) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(r->device));
    if (frame_tick(r->rp.state, r->rp.n_channels, nullptr, r->stream)) return JAERO_E_CUDA;
    r->launches++;
    return JAERO_OK;
}
int jaero_rt_read_packets(jaero_rt *r, uint8_t *out, int cap_packets, int32_t *counts)
{
    if (!r || !out || !counts || cap_packets <= 0) { set_error("jaero_rt_read_packets: bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(r->device));
    bool overflow = false;
    if (read_records(r->rp.state, r->h_state, r->rp.out, r->h_out, r->rp.n_channels, RT_OUT, RT_OUT_BYTES, r->stream,
                     out, cap_packets, counts, &overflow)) return JAERO_E_CUDA;
    if (frame_out_reset(r->rp.state, r->rp.n_channels, r->stream)) return JAERO_E_CUDA;
    r->launches++;
    if (overflow) { set_error("R/T packet queue overflow: read more often"); return JAERO_E_OVERFLOW; }
    return JAERO_OK;
}
int jaero_rt_get_stats(jaero_rt *r, int32_t *n_trials, int32_t *n_bad, int32_t *dcd)
{
    if (!r) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(r->device));
    const size_t C = r->rp.n_channels;
    JB_CUDA(cudaMemcpyAsync(r->h_state, r->rp.state, C * sizeof(RtState), cudaMemcpyDeviceToHost, r->stream));
    JB_CUDA(cudaStreamSynchronize(r->stream));
    for (size_t ch = 0; ch < C; ch++) {
        if (n_trials) n_trials[ch] = r->h_state[ch].n_trials;
        if (n_bad) n_bad[ch] = r->h_state[ch].n_bad;
        if (dcd) dcd[ch] = r->h_state[ch].datacd;
    }
    return JAERO_OK;
}

} // extern "C"

// ====================================================================== C-channel (8400 bps) frame layer (§8(f)3)
extern "C" {

int jaero_cchannel_create(int n_channels, int device, jaero_cchannel **out)
{
    if (!out || n_channels <= 0) { set_error("jaero_cchannel_create: bad argument"); return JAERO_E_ARG; }
    CreateGuard<jaero_cchannel> guard(jaero_cchannel_destroy);
    int r = guard.begin("jaero_cchannel_create", device); if (r) return r;
    jaero_cchannel *c = guard.obj;
    JB_CUDA(cudaEventCreateWithFlags(&c->ev_batch, cudaEventDisableTiming));
    JB_CUDA(cudaEventCreateWithFlags(&c->ev_own, cudaEventDisableTiming));
    CChanParams &cp = c->params;
    cp.n_channels = n_channels; cp.dl2_len = 2714 - 6 + 1;                     // dl2.setLength(2714-6) (aerol.cpp:1037)
    const size_t C = n_channels;
    int rc = 0;
    rc |= owned_alloc(c, &cp.state, C); rc |= owned_alloc(c, &cp.coded, C * CC_SLOTS * CC_CODED_PITCH); rc |= owned_alloc(c, &cp.decoded, C * CC_QUEUE * CC_DEC);
    rc |= owned_alloc(c, &cp.ready, C); rc |= owned_alloc(c, &cp.dl2, C * cp.dl2_len); rc |= owned_alloc(c, &cp.out, C * CC_OUT * CC_RECORD);
    rc |= owned_alloc(c, &c->vit_overlap, C * 64); rc |= owned_alloc(c, &c->vit_overlap_len, C); rc |= owned_alloc(c, &c->vit_renorm, C); rc |= owned_alloc(c, &c->vit_valid, C);
    if (rc) return JAERO_E_CUDA;
    if (frame_set_scrambler() || per_channel_launch(cchan_init_kernel, n_channels, c->stream, cp)) return JAERO_E_CUDA;
    JB_CUDA(cudaStreamSynchronize(c->stream));
    JB_CUDA(cudaMallocHost(&c->h_state, C * sizeof(CChanState)));
    JB_CUDA(cudaMallocHost(&c->h_out, C * CC_OUT * CC_RECORD));
    *out = guard.release();
    return JAERO_OK;
}
void jaero_cchannel_destroy(jaero_cchannel *c) { layer_destroy(c); }
int64_t jaero_cchannel_launch_count(const jaero_cchannel *c) { return c ? c->launches : 0; }

int jaero_cchannel_process_batch(jaero_cchannel *c, jaero_batch *b) { return layer_process_batch(c, b, "jaero_cchannel_process_batch"); }
int jaero_cchannel_process_softbits(jaero_cchannel *c, const int16_t *soft, size_t cap, const int32_t *counts)
{
    return layer_process_softbits(c, soft, cap, counts, "jaero_cchannel_process_softbits");
}
int jaero_cchannel_tick(jaero_cchannel *c, jaero_batch *b) { return layer_dcd_launch(c, b, -1, "jaero_cchannel_tick", frame_tick<CChanState>); }
int jaero_cchannel_lost_signal(jaero_cchannel *c, jaero_batch *b, int channel)     // AeroL::LostSignal, see jaero_pchannel_lost_signal
{
    return layer_dcd_launch(c, b, channel, "jaero_cchannel_lost_signal", frame_lost<CChanState>, channel);
}
int jaero_cchannel_write_batch(jaero_cchannel *c, jaero_batch *b, const int16_t *pcm, size_t n, size_t stride)   // see jaero_pchannel_write_batch
{
    return layer_write_batch(c, b, pcm, n, stride, "jaero_cchannel_write_batch", jaero_cchannel_process_batch);
}
int jaero_cchannel_read_frames(jaero_cchannel *c, uint8_t *out, int cap_frames, int32_t *counts)
{
    if (!c || !out || !counts || cap_frames <= 0) { set_error("jaero_cchannel_read_frames: bad argument"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(c->device));
    bool overflow = false;
    if (read_records(c->params.state, c->h_state, c->params.out, c->h_out, c->params.n_channels, CC_OUT, CC_RECORD, c->stream,
                     out, cap_frames, counts, &overflow)) return JAERO_E_CUDA;
    if (frame_out_reset(c->params.state, c->params.n_channels, c->stream)) return JAERO_E_CUDA;
    c->own_dirty = true;
    c->launches++;
    if (overflow) { set_error("C-channel frame queue overflow: read more often"); return JAERO_E_OVERFLOW; }
    return JAERO_OK;
}
int jaero_cchannel_get_stats(jaero_cchannel *c, int32_t *dcd, int64_t *su_total, int64_t *su_ok) { return layer_get_stats(c, dcd, su_total, su_ok); }

} // extern "C"

// ====================================================================== ingest router (§8(f)4, host side)
// The many-channel feed of the reference: one ZMQ PUB topic per channel, every message three frames
// [topic][uint32 sample rate][int16 PCM] (JAERO/zmq_audioreceiver.cpp:37-87, subscription = the first 5 bytes of the
// topic, :46), delivered to the demodulator's dataReceived(audio, sampleRate) slot (oqpskdemodulator.cpp:686-693).
// This router takes the three frames as the transport hands them over (no libzmq dependency), files the PCM under the
// channel whose topic matches and, once every channel has n samples, feeds them to a batch in one jaero_batch_write.
struct jaero_ingest {
    int n_channels; uint32_t rate; size_t cap;
    std::vector<std::string> topics;
    std::vector<int16_t> pcm;               // [n_channels][cap]
    std::vector<size_t> fill;
    long long dropped_bytes, messages;
};

extern "C" {

int jaero_ingest_create(int n_channels, const char *const *topics, uint32_t sample_rate, size_t capacity_samples, jaero_ingest **out)
{
    if (!out || !topics || n_channels <= 0 || capacity_samples == 0) { set_error("jaero_ingest_create: bad argument"); return JAERO_E_ARG; }
    jaero_ingest *g = new (std::nothrow) jaero_ingest();
    if (!g) { set_error("out of host memory"); return JAERO_E_ARG; }
    g->n_channels = n_channels; g->rate = sample_rate; g->cap = capacity_samples; g->dropped_bytes = 0; g->messages = 0;
    for (int c = 0; c < n_channels; c++) {
        if (!topics[c]) { delete g; set_error("jaero_ingest_create: null topic"); return JAERO_E_ARG; }
        g->topics.push_back(std::string(topics[c]).substr(0, 5));          // zmq_setsockopt(..., ZMQ_SUBSCRIBE, topic, 5)
    }
    g->pcm.assign((size_t)n_channels * capacity_samples, 0);
    g->fill.assign(n_channels, 0);
    *out = g;
    return JAERO_OK;
}
void jaero_ingest_destroy(jaero_ingest *g) { delete g; }

int jaero_ingest_message(jaero_ingest *g, const void *topic, size_t topic_len, const void *rate, size_t rate_len, const void *pcm, size_t pcm_bytes)
{
    if (!g || !topic || !rate || (!pcm && pcm_bytes)) { set_error("jaero_ingest_message: null argument"); return JAERO_E_ARG; }
    if (rate_len != 4) { set_error("jaero_ingest_message: the sample-rate frame must be 4 bytes"); return JAERO_E_ARG; }
    uint32_t r; memcpy(&r, rate, 4);                                           // memcpy(&sampleRate, rate, 4) (:70)
    int ch = -1;
    for (int c = 0; c < g->n_channels && ch < 0; c++) {
        const std::string &t = g->topics[c];
        if (topic_len >= t.size() && memcmp(topic, t.data(), t.size()) == 0) ch = c;   // prefix match, as a ZMQ subscription does
    }
    if (ch < 0) { set_error("jaero_ingest_message: no channel subscribes to this topic"); return JAERO_E_ARG; }
    if (r != g->rate) { set_error("jaero_ingest_message: sample rate differs from the batch's (the reference re-applies its settings; a batch is fixed-rate)"); return JAERO_E_STATE; }
    g->messages++;
    size_t n = pcm_bytes / 2;                                                   // writeData: len/2 int16 samples
    const size_t room = g->cap - g->fill[ch];
    // a full channel buffer refuses the whole message (nothing is filed, so the caller can flush and re-send): dropping
    // the tail silently would desynchronise this channel against the lock-step batch
    if (n > room) { g->dropped_bytes += (long long)n * 2; set_error("jaero_ingest_message: channel buffer full (flush the batch, then re-send this message)"); return JAERO_E_OVERFLOW; }
    memcpy(g->pcm.data() + (size_t)ch * g->cap + g->fill[ch], pcm, n * 2);
    g->fill[ch] += n;
    return ch;
}
size_t jaero_ingest_available(const jaero_ingest *g)
{
    if (!g) return 0;
    size_t m = g->cap;
    for (int c = 0; c < g->n_channels; c++) m = std::min(m, g->fill[c]);
    return m;
}
int jaero_ingest_flush(jaero_ingest *g, jaero_batch *b, size_t n)
{
    if (!g || !b || b->p.n_channels != g->n_channels) { set_error("jaero_ingest_flush: batch mismatch"); return JAERO_E_ARG; }
    if (n == 0) return JAERO_OK;
    if (n > jaero_ingest_available(g)) { set_error("jaero_ingest_flush: not every channel has that many samples"); return JAERO_E_STATE; }
    const int rc = jaero_batch_write(b, g->pcm.data(), n, g->cap);
    if (rc != JAERO_OK) return rc;
    JB_CUDA(cudaStreamSynchronize(b->stream));                                 // the pageable staging rows are reused below
    for (int c = 0; c < g->n_channels; c++) {
        int16_t *row = g->pcm.data() + (size_t)c * g->cap;
        memmove(row, row + n, (g->fill[c] - n) * 2);
        g->fill[c] -= n;
    }
    return JAERO_OK;
}

} // extern "C"

// ------------------------------------------------------------------ wideband IQ down-converter
// Filter design: Kaiser-windowed sinc, designed for DDC_DESIGN_DB of stopband attenuation (the specification asks 70 dB; the
// margin covers the length estimate) with its cut-off half-way through the transition band and unit gain at 0 Hz. A Kaiser
// window's passband ripple equals its stopband ripple, far inside the +-0.1 dB the specification allows.
static const double DDC_DESIGN_DB = 76.0;
static const int DDC_MAX_TAPS = 1 << 15;

// Taps for the design; max_taps + 1 when the estimate reaches max_taps
static int kaiser_length(double fs, double fpass, double fstop, int max_taps = DDC_MAX_TAPS)
{
    const double dw = 2 * M_PI * (fstop - fpass) / fs;
    const double n = (DDC_DESIGN_DB - 7.95) / (2.285 * dw) + 1.0;
    if (!(n < max_taps)) return max_taps + 1;
    return (int)ceil(n) | 1;                                        // odd: a whole-sample group delay
}
static double bessel_i0(double x)
{
    double s = 1.0, t = 1.0;
    for (int k = 1; k < 200 && t > 1e-17 * s; k++) { t *= (x / (2.0 * k)) * (x / (2.0 * k)); s += t; }
    return s;
}
static void kaiser_lowpass(double fs, double fpass, double fstop, int n, double *h)
{
    const double beta = 0.1102 * (DDC_DESIGN_DB - 8.7), fc = 0.5 * (fpass + fstop) / fs, m = 0.5 * (n - 1);
    double sum = 0.0;
    for (int k = 0; k < n; k++) {
        const double t = k - m, r = m > 0 ? t / m : 0.0;
        const double sinc = t == 0.0 ? 2 * fc : sin(2 * M_PI * fc * t) / (M_PI * t);
        h[k] = sinc * bessel_i0(beta * sqrt(std::max(0.0, 1.0 - r * r))) / bessel_i0(beta);
        sum += h[k];
    }
    for (int k = 0; k < n; k++) h[k] /= sum;
}

static const int DDC_MAX_INTERPOLATION = 256;

struct DdcPlan { int L, D1, K1, D2, K2; double fs1; };

// The split M = D1 * D2 with the fewest multiply-adds per output: 8 (D2 / L) K1 + 4 ceil(K2 / L) flop (a stage-1 tap is a
// complex x complex product, twice a stage-2 tap, and of the K2 stage-2 taps only every L-th meets a sample that is not a
// stuffed zero). The search compares that count times L / 4, an integer. Stage 1 passes B/2 and stops Fs1 - B/2 - transition,
// everything that would alias into stage 2's passband; stage 2, at L * Fs1, passes B/2 and stops B/2 + transition, which also
// removes the images of the x L zero-stuffing. For L = 1 a single stage (D2 = 1, h2 = {1}) is a candidate and a stage 1 that
// does not decimate is not; for L > 1 stage 2 always interpolates, so every divisor D1 of M is a candidate.
static int ddc_plan_stages(double fs, int L, int M, double B, double dT, DdcPlan *out, const char *fn)
{
    const double fs_out = fs * L / M, fp = 0.5 * B, fst = 0.5 * B + dT;
    if (!(fs > 0) || M < 1 || !(B > 0) || !(dT > 0)) { set_error(std::string(fn) + ": rates, bandwidth and transition must be positive"); return JAERO_E_ARG; }
    if (L < 1 || L > DDC_MAX_INTERPOLATION) { set_error(std::string(fn) + ": interpolation must be 1 to " + std::to_string(DDC_MAX_INTERPOLATION)); return JAERO_E_ARG; }
    if (std::gcd(L, M) != 1) { set_error(std::string(fn) + ": interpolation and decimation have a common factor; reduce the ratio L/M"); return JAERO_E_ARG; }
    if (!(fst <= 0.5 * fs_out)) { set_error(std::string(fn) + ": bandwidth/2 + transition must not exceed half the output rate"); return JAERO_E_ARG; }
    long best = -1;
    for (int D1 = 1; D1 <= M; D1++) {
        if (M % D1) continue;
        DdcPlan c{L, D1, 0, M / D1, 1, fs / D1};
        if (L == 1 && c.D2 == 1) c.K1 = kaiser_length(fs, fp, fst);
        else {
            if (L == 1 && D1 == 1) continue;                         // a stage 1 that does not decimate only adds work
            if (!(c.fs1 - fst > fp)) continue;                       // stage 1's output rate leaves it no stopband
            c.K1 = kaiser_length(fs, fp, c.fs1 - fst);
            c.K2 = kaiser_length(c.fs1 * L, fp, fst);
        }
        if (c.K1 > DDC_MAX_TAPS || c.K2 > DDC_MAX_TAPS || (DDC_TILE_J - 1) * D1 + c.K1 > DDC_MAX_TILE) continue;
        const long cost = 2L * c.D2 * c.K1 + (long)L * ((c.K2 + L - 1) / L);
        if (best < 0 || cost < best) { best = cost; *out = c; }
    }
    if (best < 0) { set_error(std::string(fn) + ": no two-stage split of this decimation meets the filter specification within the tap limits"); return JAERO_E_ARG; }
    return JAERO_OK;
}
// h2 sums to L: the zero-stuffing divides the signal's level by L, so the passband gain is 1.
static void ddc_design(double fs, double B, double dT, const DdcPlan &c, double *h1, double *h2)
{
    const double fp = 0.5 * B, fst = 0.5 * B + dT;
    if (c.L == 1 && c.D2 == 1) { kaiser_lowpass(fs, fp, fst, c.K1, h1); h2[0] = 1.0; return; }
    kaiser_lowpass(fs, fp, c.fs1 - fst, c.K1, h1);
    kaiser_lowpass(c.fs1 * c.L, fp, fst, c.K2, h2);
    if (c.L > 1)
        for (int k = 0; k < c.K2; k++) h2[k] *= c.L;
}
// round(f / fs * 2^32) mod 2^32
static uint32_t tuning_word(double f, double fs) { return (uint32_t)(uint64_t)llround(f / fs * 4294967296.0); }

// ------------------------------------------------------------------ host plumbing of the front-end stages
// What the down-converter, the rate converter, the scanner and the identifier share: a device and a stream that set_stream can
// replace, owned buffers, and the samples (per channel) taken and kernels launched since create.
struct Stage {
    int device; cudaStream_t stream, own_stream;
    std::vector<void *> allocs;
    long long n_in, launches;
};
// The down-converter's and the rate converter's output: the [n_channels][pcm_stride] PCM rows of the last write
struct PcmStage : Stage {
    int16_t *d_pcm; size_t pcm_cap, pcm_n, pcm_stride;
};

// The whole of a stage's destroy, for a non-null o: its queued work drains, then everything it owns is freed
template <class O> void destroy_stage(O *o, std::initializer_list<void *> grown)
{
    cudaSetDevice(o->device);
    cudaStreamSynchronize(o->stream);
    release(o, grown, {}, o->own_stream);
}

static const size_t MAX_WRITE_SAMPLES = (size_t)1 << 34;
static int arg_error(const char *fn, const char *what) { set_error(std::string(fn) + ": " + what); return JAERO_E_ARG; }
static size_t iq_sample_bytes(int format) { return format == JAERO_IQ_CU8 ? 2 : 4; }

// Argument checks of an IQ write, in this order: null handle or buffer, format, alignment to one sample (device buffers only), length
static int iq_write_args(const void *o, const void *iq, size_t n, int format, bool device, const char *fn)
{
    if (!o || !iq) return arg_error(fn, "null argument");
    if (format != JAERO_IQ_CU8 && format != JAERO_IQ_CS16) return arg_error(fn, "unknown IQ format");
    if (device && ((uintptr_t)iq & (iq_sample_bytes(format) - 1))) return arg_error(fn, "IQ pointer not aligned to one sample");
    if (n > MAX_WRITE_SAMPLES) return arg_error(fn, "too many samples in one write");
    return JAERO_OK;
}
// Argument checks of a [n_channels][stride] PCM write, in this order: null handle or buffer, alignment to one sample (device
// buffers only), stride, length
static int pcm_write_args(const void *o, const int16_t *pcm, size_t n, size_t stride, bool device, const char *fn)
{
    if (!o || !pcm) return arg_error(fn, "null argument");
    if (device && ((uintptr_t)pcm & 1)) return arg_error(fn, "PCM pointer not aligned to one sample");
    if (stride < n) return arg_error(fn, "channel stride is smaller than n_samples");
    if (n > MAX_WRITE_SAMPLES) return arg_error(fn, "too many samples in one write");
    return JAERO_OK;
}

// A host IQ write: the bytes are staged in o->d_raw, then written as from the device. The copy is waited for, so the caller may
// reuse its pageable buffer on return.
template <class O> int stage_iq_write(O *o, const void *iq, size_t n, int format, const char *fn, int (*write_device)(O *, const void *, size_t, int))
{
    int r = iq_write_args(o, iq, n, format, false, fn); if (r) return r;
    JB_CUDA(cudaSetDevice(o->device));
    const size_t bytes = n * iq_sample_bytes(format);
    if (grow((uint8_t **)&o->d_raw, &o->raw_cap, std::max<size_t>(bytes, 4), o->stream)) return JAERO_E_CUDA;
    if (bytes) {
        JB_CUDA(cudaMemcpyAsync(o->d_raw, iq, bytes, cudaMemcpyHostToDevice, o->stream));
        JB_CUDA(cudaStreamSynchronize(o->stream));
    }
    return write_device(o, o->d_raw, n, format);
}
// A host PCM write: the rows are staged densely in o->d_in, [n_channels][n], then written as from the device, as above
template <class O> int stage_pcm_write(O *o, const int16_t *pcm, size_t n, size_t stride, const char *fn,
                                       int (*write_device)(O *, const int16_t *, size_t, size_t))
{
    int r = pcm_write_args(o, pcm, n, stride, false, fn); if (r) return r;
    JB_CUDA(cudaSetDevice(o->device));
    const size_t C = (size_t)o->p.n_channels;
    if (grow(&o->d_in, &o->in_cap, std::max<size_t>(C * n, 1), o->stream)) return JAERO_E_CUDA;
    if (n) {
        JB_CUDA(cudaMemcpy2DAsync(o->d_in, n * sizeof(int16_t), pcm, stride * sizeof(int16_t), n * sizeof(int16_t), C, cudaMemcpyHostToDevice,
                                  o->stream));
        JB_CUDA(cudaStreamSynchronize(o->stream));
    }
    return write_device(o, o->d_in, n, n);
}

// Outputs m of an L/D rate change with floor(m D / L) in [n0, n0 + n): ceil((n0 + n) L / D) - ceil(n0 L / D)
static size_t rational_outputs(long long n0, long long n, long long L, long long D) { return (size_t)(((n0 + n) * L + D - 1) / D - (n0 * L + D - 1) / D); }
// 16-byte output rows: jaero_batch_write_device reads them in place
static size_t pcm_row_stride(size_t m) { return std::max<size_t>(8, (m + 7) & ~(size_t)7); }

// [L][R] per-phase taps of a K-tap prototype, hp[phi][r] = h[phi + r L], zero past its end
static std::vector<double> polyphase_fold(const double *h, int K, int L, int R)
{
    std::vector<double> hp((size_t)L * R, 0.0);
    for (int k = 0; k < K; k++) hp[(size_t)(k % L) * R + k / L] = h[k];
    return hp;
}

template <class O> int pcm_output(O *o, const int16_t **d_pcm, size_t *n, size_t *stride, const char *fn)
{
    if (!o || !d_pcm || !n || !stride) return arg_error(fn, "null argument");
    *d_pcm = o->d_pcm; *n = o->pcm_n; *stride = o->pcm_stride;
    return JAERO_OK;
}
template <class O> int pcm_read(O *o, int16_t *out, size_t cap, size_t *n, const char *fn)
{
    if (!o || !out || !n) return arg_error(fn, "null argument");
    if (cap < o->pcm_n) return arg_error(fn, "cap_per_channel is smaller than the last write's output");
    JB_CUDA(cudaSetDevice(o->device));
    if (o->pcm_n)
        JB_CUDA(cudaMemcpy2DAsync(out, cap * sizeof(int16_t), o->d_pcm, o->pcm_stride * sizeof(int16_t), o->pcm_n * sizeof(int16_t),
                                  o->p.n_channels, cudaMemcpyDeviceToHost, o->stream));
    JB_CUDA(cudaStreamSynchronize(o->stream));
    *n = o->pcm_n;
    return JAERO_OK;
}
template <class O> int pcm_stats(O *o, int64_t *inputs, int64_t *clipped)
{
    if (!o) { set_error("null handle"); return JAERO_E_ARG; }
    if (inputs) *inputs = o->n_in;
    if (clipped) {
        JB_CUDA(cudaSetDevice(o->device));
        JB_CUDA(cudaMemcpyAsync(clipped, o->p.clipped, o->p.n_channels * sizeof(int64_t), cudaMemcpyDeviceToHost, o->stream));
        JB_CUDA(cudaStreamSynchronize(o->stream));
    }
    return JAERO_OK;
}

// nfft of the scanner (max_nfft 65536) and the identifier (16384): a power of two from 1024
static bool pow2_nfft(int nfft, int max_nfft) { return nfft >= 1024 && nfft <= max_nfft && (nfft & (nfft - 1)) == 0; }

// The tables of a windowed four-step FFT of nfft points, in two owned buffers: the n1 x n2 split (n1 = 2^floor(log2(nfft) / 2)),
// the twiddles W_N^k and the periodic Hann window. Returns the window's sum of squares in *wss.
template <class O, class P> int four_step_tables(O *o, P &p, int nfft, double *wss)
{
    int lg = 0;
    while ((1 << lg) < nfft) lg++;
    p.n1 = 1 << (lg / 2); p.n2 = nfft / p.n1;
    const std::vector<std::complex<double>> tw = twiddles(nfft);
    std::vector<double> win(nfft);
    *wss = 0.0;
    for (int k = 0; k < nfft; k++) {
        win[k] = 0.5 - 0.5 * tw[k].real();
        *wss += win[k] * win[k];
    }
    double2 *dtw; double *dwin;
    if (owned_alloc(o, &dtw, (size_t)nfft) || owned_alloc(o, &dwin, (size_t)nfft)) return JAERO_E_CUDA;
    p.tw = dtw; p.win = dwin;
    JB_CUDA(cudaMemcpyAsync(dtw, tw.data(), nfft * sizeof(double2), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaMemcpyAsync(dwin, win.data(), nfft * sizeof(double), cudaMemcpyHostToDevice, o->stream));
    JB_CUDA(cudaStreamSynchronize(o->stream));                       // the tables are in place, the host vectors may go
    return JAERO_OK;
}

// The frames a write of n samples completes, for a stage that has taken n_in samples and completed `frames` frames of N samples
// every hop. The write's samples and the carry sit at x0 + j: the carry is the n_in - x0 samples from the first incomplete frame.
struct FrameSpan {
    long long total, x0, carry, f_end, F, x1;                       // x1: the first sample an incomplete frame needs after the write
};
static FrameSpan frame_span(long long n_in, long long frames, long long N, long long hop, size_t n)
{
    FrameSpan s;
    s.total = n_in + (long long)n;
    s.x0 = frames * hop; s.carry = n_in - s.x0;
    s.f_end = s.total >= N ? (s.total - N) / hop + 1 : 0; s.F = s.f_end - frames;
    s.x1 = s.f_end * hop;
    return s;
}

struct jaero_ddc : PcmStage {
    DdcParams p;
    double fs_in, fs_out, B;
    std::vector<double> h1;                                          // host copy, for re-folding on set_offset
    std::vector<uint32_t> T, S;
    std::vector<double2> h1c;                                        // [K1][cpad] staging for the folded taps
    void *d_raw; size_t raw_cap;                                     // host writes: the IQ bytes staged on the device
    double2 *d_x, *d_u; size_t x_cap, u_cap;
};

// Retunes are ordered on the DDC's stream like its kernels: writes queued before a retune read the old values, writes after it the
// new ones, with no wait on the host. A pageable host-to-device cudaMemcpyAsync has copied its source out of the host buffer
// when it returns (CUDA runtime API synchronisation rules), so the host tables may change again right after.
// The tuning words of channel c (c < 0: every channel), host words -> device words.
static int ddc_upload_words(jaero_ddc *d, const std::vector<uint32_t> &w, const uint32_t *dev, int c)
{
    const size_t c0 = c < 0 ? 0 : (size_t)c, n = c < 0 ? (size_t)d->p.n_channels : 1;
    JB_CUDA(cudaMemcpyAsync((void *)(dev + c0), w.data() + c0, n * sizeof(uint32_t), cudaMemcpyHostToDevice, d->stream));
    return JAERO_OK;
}
// Folds channel c's mix into its stage-1 taps (c < 0: every channel) and uploads that channel's column of the [K1][cpad] table
// with its tuning word.
static int ddc_upload_offset(jaero_ddc *d, int c)
{
    DdcParams &p = d->p;
    const int c0 = c < 0 ? 0 : c, c1 = c < 0 ? p.n_channels : c + 1;
    for (int ch = c0; ch < c1; ch++)
        for (int k = 0; k < p.K1; k++) {
            const double th = 2 * M_PI * (double)(uint32_t)((uint32_t)k * d->T[ch]) / 4294967296.0;
            d->h1c[(size_t)k * p.cpad + ch] = make_double2(d->h1[k] * cos(th), d->h1[k] * sin(th));
        }
    const size_t pitch = (size_t)p.cpad * sizeof(double2);
    if (c < 0) JB_CUDA(cudaMemcpyAsync((void *)p.h1c, d->h1c.data(), d->h1c.size() * sizeof(double2), cudaMemcpyHostToDevice, d->stream));
    else JB_CUDA(cudaMemcpy2DAsync((void *)(p.h1c + c), pitch, d->h1c.data() + c, pitch, sizeof(double2), p.K1, cudaMemcpyHostToDevice, d->stream));
    return ddc_upload_words(d, d->T, p.T, c);
}
static bool ddc_offset_ok(const jaero_ddc *d, double hz) { return std::isfinite(hz) && fabs(hz) <= 0.5 * d->fs_in - 0.5 * d->B; }
static bool ddc_audio_ok(const jaero_ddc *d, double hz) { return std::isfinite(hz) && hz - 0.5 * d->B > 0 && hz + 0.5 * d->B < 0.5 * d->fs_out; }

extern "C" {

// jaero_ddc_plan and jaero_ddc_plan_rational: stages receives {D1, K1, D2, K2}, preceded by L when with_l
static int ddc_plan_query(double input_rate, int L, int M, double bandwidth, double transition, int32_t *stages, bool with_l, double *h1,
                          double *h2, const char *fn)
{
    if (!stages) { set_error(std::string(fn) + ": null argument"); return JAERO_E_ARG; }
    DdcPlan c;
    const int r = ddc_plan_stages(input_rate, L, M, bandwidth, transition, &c, fn);
    if (r) return r;
    if (with_l) *stages++ = c.L;
    stages[0] = c.D1; stages[1] = c.K1; stages[2] = c.D2; stages[3] = c.K2;
    if (h1 && h2) ddc_design(input_rate, bandwidth, transition, c, h1, h2);
    else if (h1 || h2) {
        std::vector<double> a(c.K1), b(c.K2);
        ddc_design(input_rate, bandwidth, transition, c, a.data(), b.data());
        if (h1) std::copy(a.begin(), a.end(), h1);
        if (h2) std::copy(b.begin(), b.end(), h2);
    }
    return JAERO_OK;
}

static int ddc_create(double input_rate, int L, int M, int n_channels, const double *offset_hz, const double *audio_hz, double bandwidth,
                      double transition, double gain, int device, jaero_ddc **out, const char *fn)
{
    const std::string f(fn);
    if (!out || n_channels <= 0 || !offset_hz || !audio_hz || !std::isfinite(gain)) { set_error(f + ": bad argument"); return JAERO_E_ARG; }
    DdcPlan c;
    { const int r = ddc_plan_stages(input_rate, L, M, bandwidth, transition, &c, fn); if (r) return r; }
    const double fs_out = input_rate * L / M;
    for (int ch = 0; ch < n_channels; ch++) {
        if (!(std::isfinite(offset_hz[ch]) && fabs(offset_hz[ch]) <= 0.5 * input_rate - 0.5 * bandwidth)) {
            set_error(f + ": channel " + std::to_string(ch) + ": |offset| must not exceed input_rate/2 - bandwidth/2"); return JAERO_E_ARG; }
        if (!(std::isfinite(audio_hz[ch]) && audio_hz[ch] - 0.5 * bandwidth > 0 && audio_hz[ch] + 0.5 * bandwidth < 0.5 * fs_out)) {
            set_error(f + ": channel " + std::to_string(ch) + ": the audio passband must lie inside (0, output_rate/2)"); return JAERO_E_ARG; }
    }
    CreateGuard<jaero_ddc> guard(jaero_ddc_destroy);
    { const int e = guard.begin(fn, device); if (e) return e; }
    jaero_ddc *d = guard.obj;
    d->own_stream = d->stream;
    d->fs_in = input_rate; d->fs_out = fs_out; d->B = bandwidth;
    DdcParams &p = d->p;
    p.n_channels = n_channels; p.cpad = (n_channels + 31) & ~31;
    p.L = c.L; p.D1 = c.D1; p.K1 = c.K1; p.D2 = c.D2; p.K2 = c.K2;
    p.R = (c.K2 + c.L - 1) / c.L;
    // the first output of a write reads back R - 1 rows from q >= j_lo - 1 (L > 1) or K2 - 1 rows from q >= j_lo (L = 1)
    p.H2 = c.L == 1 ? c.K2 - 1 : p.R;
    p.scale = gain * 32768.0;
    d->h1.resize(c.K1);
    std::vector<double> h2(c.K2);
    ddc_design(input_rate, bandwidth, transition, c, d->h1.data(), h2.data());
    const std::vector<double> h2p = polyphase_fold(h2.data(), c.K2, c.L, p.R);
    d->T.resize(n_channels); d->S.resize(n_channels);
    for (int ch = 0; ch < n_channels; ch++) { d->T[ch] = tuning_word(offset_hz[ch], input_rate); d->S[ch] = tuning_word(audio_hz[ch], fs_out); }
    d->h1c.assign((size_t)c.K1 * p.cpad, make_double2(0.0, 0.0));
    const size_t cp = p.cpad;
    double2 *h1c; double *dh2; uint32_t *T, *S;
    int rc = 0;
    rc |= owned_alloc(d, &h1c, (size_t)c.K1 * cp); rc |= owned_alloc(d, &dh2, h2p.size());
    rc |= owned_alloc(d, &T, cp); rc |= owned_alloc(d, &S, cp);
    rc |= owned_alloc(d, &p.xhist, (size_t)std::max(1, c.K1 - 1)); rc |= owned_alloc(d, &p.uhist, (size_t)std::max(1, p.H2) * cp);
    rc |= owned_alloc(d, &p.clipped, cp);
    if (rc) return JAERO_E_CUDA;
    p.h1c = h1c; p.h2 = dh2; p.T = T; p.S = S;
    JB_CUDA(cudaMemcpyAsync(dh2, h2p.data(), h2p.size() * sizeof(double), cudaMemcpyHostToDevice, d->stream));
    if (ddc_upload_offset(d, -1) || ddc_upload_words(d, d->S, p.S, -1)) return JAERO_E_CUDA;
    JB_CUDA(cudaStreamSynchronize(d->stream));                       // the zeroed histories and the tables are in place
    *out = guard.release();
    return JAERO_OK;
}

int jaero_ddc_plan(double input_rate, int decimation, double bandwidth, double transition, int32_t stages[4], double *h1, double *h2)
{
    return ddc_plan_query(input_rate, 1, decimation, bandwidth, transition, stages, false, h1, h2, "jaero_ddc_plan");
}
int jaero_ddc_plan_rational(double input_rate, int interpolation, int decimation, double bandwidth, double transition, int32_t stages[5],
                            double *h1, double *h2)
{
    return ddc_plan_query(input_rate, interpolation, decimation, bandwidth, transition, stages, true, h1, h2, "jaero_ddc_plan_rational");
}
int jaero_ddc_create(double input_rate, int decimation, int n_channels, const double *offset_hz, const double *audio_hz, double bandwidth,
                     double transition, double gain, int device, jaero_ddc **out)
{
    return ddc_create(input_rate, 1, decimation, n_channels, offset_hz, audio_hz, bandwidth, transition, gain, device, out, "jaero_ddc_create");
}
int jaero_ddc_create_rational(double input_rate, int interpolation, int decimation, int n_channels, const double *offset_hz,
                              const double *audio_hz, double bandwidth, double transition, double gain, int device, jaero_ddc **out)
{
    return ddc_create(input_rate, interpolation, decimation, n_channels, offset_hz, audio_hz, bandwidth, transition, gain, device, out,
                      "jaero_ddc_create_rational");
}
void jaero_ddc_destroy(jaero_ddc *d) { if (d) destroy_stage(d, {d->d_raw, d->d_x, d->d_u, d->d_pcm}); }
int64_t jaero_ddc_launch_count(const jaero_ddc *d) { return d ? d->launches : 0; }

int jaero_ddc_write_device(jaero_ddc *d, const void *d_iq, size_t n, int format)
{
    int r = iq_write_args(d, d_iq, n, format, true, "jaero_ddc_write_device"); if (r) return r;
    JB_CUDA(cudaSetDevice(d->device));
    DdcParams &p = d->p;
    const long long n0 = d->n_in;
    const size_t M = rational_outputs(n0, (long long)n, p.L, (long long)p.D1 * p.D2), J = rational_outputs(n0, (long long)n, 1, p.D1);
    const size_t stride = pcm_row_stride(M);
    if (n > 0) {
        // a failed write leaves the output of the previous one described
        if (grow(&d->d_x, &d->x_cap, (size_t)(p.K1 - 1) + n, d->stream) || grow(&d->d_u, &d->u_cap, ((size_t)p.H2 + J) * p.cpad, d->stream) ||
            grow(&d->d_pcm, &d->pcm_cap, (size_t)p.n_channels * stride, d->stream)) return JAERO_E_CUDA;
        if (ddc_run(p, d_iq, format, n0, (long long)n, d->d_x, d->d_u, d->d_pcm, stride, d->stream, &d->launches)) return JAERO_E_CUDA;
        d->n_in += (long long)n;
    }
    d->pcm_n = M; d->pcm_stride = stride;
    return JAERO_OK;
}
int jaero_ddc_write(jaero_ddc *d, const void *iq, size_t n, int format) { return stage_iq_write(d, iq, n, format, "jaero_ddc_write", jaero_ddc_write_device); }
int jaero_ddc_output(jaero_ddc *d, const int16_t **d_pcm, size_t *n, size_t *stride) { return pcm_output(d, d_pcm, n, stride, "jaero_ddc_output"); }
int jaero_ddc_read_pcm(jaero_ddc *d, int16_t *out, size_t cap, size_t *n) { return pcm_read(d, out, cap, n, "jaero_ddc_read_pcm"); }
int jaero_ddc_set_stream(jaero_ddc *d, void *cuda_stream) { return switch_stream(d, cuda_stream); }
int jaero_ddc_set_offset(jaero_ddc *d, int channel, double hz)
{
    if (!d || channel < -1 || channel >= d->p.n_channels) { set_error("jaero_ddc_set_offset: bad argument"); return JAERO_E_ARG; }
    if (!ddc_offset_ok(d, hz)) { set_error("jaero_ddc_set_offset: |offset| must not exceed input_rate/2 - bandwidth/2"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(d->device));
    const uint32_t w = tuning_word(hz, d->fs_in);
    for (int c = 0; c < d->p.n_channels; c++) if (channel < 0 || c == channel) d->T[c] = w;
    return ddc_upload_offset(d, channel);
}
int jaero_ddc_set_audio_freq(jaero_ddc *d, int channel, double hz)
{
    if (!d || channel < -1 || channel >= d->p.n_channels) { set_error("jaero_ddc_set_audio_freq: bad argument"); return JAERO_E_ARG; }
    if (!ddc_audio_ok(d, hz)) { set_error("jaero_ddc_set_audio_freq: the audio passband must lie inside (0, output_rate/2)"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(d->device));
    const uint32_t w = tuning_word(hz, d->fs_out);
    for (int c = 0; c < d->p.n_channels; c++) if (channel < 0 || c == channel) d->S[c] = w;
    return ddc_upload_words(d, d->S, d->p.S, channel);
}
int jaero_ddc_get_stats(jaero_ddc *d, int64_t *inputs, int64_t *clipped) { return pcm_stats(d, inputs, clipped); }

} // extern "C"

// ------------------------------------------------------------------ PCM rate converter
// One Kaiser low-pass prototype at L * input_rate, designed as the down-converter's stages are: it passes [0, passband_hz] and
// stops from min(input_rate, output_rate)/2, which removes both the aliases of the decimation and the images of the x L
// zero-stuffing. 11025 -> 48000 Hz is L = 640 and about 61000 taps, hence limits above the down-converter's.
static const int RESAMPLE_MAX_RATIO = 1024;
static const int RESAMPLE_MAX_TAPS = 1 << 17;

struct ResamplePlan { int L, M, K; double fs_up, fpass, fstop; };

static int resample_plan_stages(double fs_in, double fs_out, double passband, ResamplePlan *out, const char *fn)
{
    const std::string f(fn);
    for (double r : {fs_in, fs_out})
        if (!(std::isfinite(r) && r >= 1 && r <= 2147483647.0 && r == floor(r))) { set_error(f + ": rates must be positive whole hertz"); return JAERO_E_ARG; }
    const long long a = (long long)fs_in, b = (long long)fs_out, g = std::gcd(a, b);
    const long long L = b / g, M = a / g;
    if (L == 1 && M == 1) { set_error(f + ": input and output rates are equal; there is nothing to resample"); return JAERO_E_ARG; }
    if (L > RESAMPLE_MAX_RATIO || M > RESAMPLE_MAX_RATIO) {
        set_error(f + ": output_rate/input_rate reduces to " + std::to_string(L) + "/" + std::to_string(M) + "; L and M must not exceed " +
                  std::to_string(RESAMPLE_MAX_RATIO));
        return JAERO_E_ARG;
    }
    const double fstop = 0.5 * (double)std::min(a, b);
    if (!(passband > 0 && passband < fstop)) { set_error(f + ": passband_hz must lie in (0, min(input_rate, output_rate)/2)"); return JAERO_E_ARG; }
    ResamplePlan c{(int)L, (int)M, 0, (double)L * fs_in, passband, fstop};
    c.K = kaiser_length(c.fs_up, passband, fstop, RESAMPLE_MAX_TAPS);
    if (c.K > RESAMPLE_MAX_TAPS) {
        set_error(f + ": the filter would need more than " + std::to_string(RESAMPLE_MAX_TAPS) + " taps; lower passband_hz"); return JAERO_E_ARG; }
    *out = c;
    return JAERO_OK;
}
// h sums to L: the zero-stuffing divides the signal's level by L, so the passband gain is 1.
static void resample_design(const ResamplePlan &c, double *h)
{
    kaiser_lowpass(c.fs_up, c.fpass, c.fstop, c.K, h);
    for (int k = 0; k < c.K; k++) h[k] *= c.L;
}

struct jaero_resample : PcmStage {
    ResampleParams p;
    int16_t *d_in; size_t in_cap;                                    // host writes: the PCM staged on the device, [C][n]
    double *d_x; size_t x_cap;                                       // [H + n][cpad] rows of the current write
};

extern "C" {

int jaero_resample_plan(double input_rate, double output_rate, double passband_hz, int32_t stages[3], double *h)
{
    if (!stages) { set_error("jaero_resample_plan: null argument"); return JAERO_E_ARG; }
    ResamplePlan c;
    const int r = resample_plan_stages(input_rate, output_rate, passband_hz, &c, "jaero_resample_plan");
    if (r) return r;
    stages[0] = c.L; stages[1] = c.M; stages[2] = c.K;
    if (h) resample_design(c, h);
    return JAERO_OK;
}

int jaero_resample_create(double input_rate, double output_rate, int n_channels, double passband_hz, int device, jaero_resample **out)
{
    const char *fn = "jaero_resample_create";
    if (!out || n_channels <= 0) { set_error(std::string(fn) + ": bad argument"); return JAERO_E_ARG; }
    ResamplePlan c;
    { const int r = resample_plan_stages(input_rate, output_rate, passband_hz, &c, fn); if (r) return r; }
    CreateGuard<jaero_resample> guard(jaero_resample_destroy);
    { const int e = guard.begin(fn, device); if (e) return e; }
    jaero_resample *s = guard.obj;
    s->own_stream = s->stream;
    ResampleParams &p = s->p;
    p.n_channels = n_channels; p.cpad = (n_channels + 31) & ~31;
    p.L = c.L; p.M = c.M; p.K = c.K;
    p.R = (c.K + c.L - 1) / c.L;
    p.H = p.R;                                                       // the first output of a write reads back R - 1 rows
    std::vector<double> h(c.K);
    resample_design(c, h.data());
    const std::vector<double> hp = polyphase_fold(h.data(), c.K, c.L, p.R);
    double *dhp;
    int rc = 0;
    rc |= owned_alloc(s, &dhp, hp.size());
    rc |= owned_alloc(s, &p.hist, (size_t)p.H * p.cpad);
    rc |= owned_alloc(s, &p.clipped, (size_t)p.cpad);
    if (rc) return JAERO_E_CUDA;
    p.hp = dhp;
    JB_CUDA(cudaMemcpyAsync(dhp, hp.data(), hp.size() * sizeof(double), cudaMemcpyHostToDevice, s->stream));
    JB_CUDA(cudaStreamSynchronize(s->stream));                       // the zeroed history and the table are in place
    *out = guard.release();
    return JAERO_OK;
}
void jaero_resample_destroy(jaero_resample *s) { if (s) destroy_stage(s, {s->d_in, s->d_x, s->d_pcm}); }
int64_t jaero_resample_launch_count(const jaero_resample *s) { return s ? s->launches : 0; }

int jaero_resample_write_device(jaero_resample *s, const int16_t *d_pcm, size_t n, size_t stride)
{
    int r = pcm_write_args(s, d_pcm, n, stride, true, "jaero_resample_write_device"); if (r) return r;
    JB_CUDA(cudaSetDevice(s->device));
    const ResampleParams &p = s->p;
    const long long n0 = s->n_in;
    const size_t M_out = rational_outputs(n0, (long long)n, p.L, p.M);
    const size_t out_stride = pcm_row_stride(M_out);
    if (n > 0) {
        // a failed write leaves the output of the previous one described
        if (grow(&s->d_x, &s->x_cap, ((size_t)p.H + n) * p.cpad, s->stream) ||
            grow(&s->d_pcm, &s->pcm_cap, (size_t)p.n_channels * out_stride, s->stream)) return JAERO_E_CUDA;
        if (resample_run(p, d_pcm, stride, n0, (long long)n, s->d_x, s->d_pcm, out_stride, s->stream, &s->launches)) return JAERO_E_CUDA;
        s->n_in += (long long)n;
    }
    s->pcm_n = M_out; s->pcm_stride = out_stride;
    return JAERO_OK;
}
int jaero_resample_write(jaero_resample *s, const int16_t *pcm, size_t n, size_t stride)
{
    return stage_pcm_write(s, pcm, n, stride, "jaero_resample_write", jaero_resample_write_device);
}
int jaero_resample_output(jaero_resample *s, const int16_t **d_pcm, size_t *n, size_t *stride)
{
    return pcm_output(s, d_pcm, n, stride, "jaero_resample_output");
}
int jaero_resample_read_pcm(jaero_resample *s, int16_t *out, size_t cap, size_t *n) { return pcm_read(s, out, cap, n, "jaero_resample_read_pcm"); }
int jaero_resample_set_stream(jaero_resample *s, void *cuda_stream) { return switch_stream(s, cuda_stream); }
int jaero_resample_get_stats(jaero_resample *s, int64_t *inputs, int64_t *clipped) { return pcm_stats(s, inputs, clipped); }

} // extern "C"

// ------------------------------------------------------------------ wideband carrier scanner
struct jaero_scan : Stage {
    ScanPlan p;
    long long frames;                                                // complete frames since create / reset (n_in: samples)
    double2 *d_carry;                                                // [nfft] samples frames * hop .. n_in - 1 (fewer than nfft)
    void *d_raw; size_t raw_cap;                                     // host writes: the IQ bytes staged on the device
    double2 *d_x, *d_work; double *d_pw; size_t x_cap, work_cap, pw_cap;
};

extern "C" {

int jaero_scan_create(double input_rate, int nfft, int hop, int device, jaero_scan **out)
{
    if (!out) { set_error("jaero_scan_create: null argument"); return JAERO_E_ARG; }
    if (!pow2_nfft(nfft, 65536)) { set_error("jaero_scan_create: nfft must be a power of two from 1024 to 65536"); return JAERO_E_ARG; }
    if (hop < 1 || hop > nfft) { set_error("jaero_scan_create: hop must be in [1, nfft]"); return JAERO_E_ARG; }
    if (!(input_rate > 0) || !std::isfinite(input_rate)) { set_error("jaero_scan_create: input_rate must be positive"); return JAERO_E_ARG; }
    CreateGuard<jaero_scan> guard(jaero_scan_destroy);
    { const int e = guard.begin("jaero_scan_create", device); if (e) return e; }
    jaero_scan *s = guard.obj;
    s->own_stream = s->stream;
    ScanPlan &p = s->p;
    p.nfft = nfft; p.hop = hop;
    int rc = 0;
    rc |= owned_alloc(s, &p.sum, (size_t)nfft); rc |= owned_alloc(s, &p.maxh, (size_t)nfft);
    rc |= owned_alloc(s, &s->d_carry, (size_t)nfft);
    if (rc) return JAERO_E_CUDA;
    double wss;
    if ((rc = four_step_tables(s, p, nfft, &wss))) return rc;
    p.inv_wss = 1.0 / wss;
    *out = guard.release();
    return JAERO_OK;
}
void jaero_scan_destroy(jaero_scan *s) { if (s) destroy_stage(s, {s->d_raw, s->d_x, s->d_work, s->d_pw}); }
int64_t jaero_scan_launch_count(const jaero_scan *s) { return s ? s->launches : 0; }

int jaero_scan_write_device(jaero_scan *s, const void *d_iq, size_t n, int format)
{
    int r = iq_write_args(s, d_iq, n, format, true, "jaero_scan_write_device"); if (r) return r;
    if (n == 0) return JAERO_OK;
    JB_CUDA(cudaSetDevice(s->device));
    const ScanPlan &p = s->p;
    const long long N = p.nfft;
    const FrameSpan w = frame_span(s->n_in, s->frames, N, p.hop, n);
    const int G = (int)std::max<long long>(1, SCAN_PASS_ELEMS / N);
    const size_t g = (size_t)std::min<long long>(std::max<long long>(w.F, 1), G);
    // every buffer is in place before anything is queued: a failed write leaves the average unchanged
    if (grow(&s->d_x, &s->x_cap, (size_t)(w.carry + (long long)n), s->stream) || grow(&s->d_work, &s->work_cap, g * N, s->stream) ||
        grow(&s->d_pw, &s->pw_cap, g * N, s->stream)) return JAERO_E_CUDA;
    if (w.carry) JB_CUDA(cudaMemcpyAsync(s->d_x, s->d_carry, w.carry * sizeof(double2), cudaMemcpyDeviceToDevice, s->stream));
    if (scan_convert(d_iq, format, (long long)n, s->d_x + w.carry, s->stream, &s->launches)) return JAERO_E_CUDA;
    if (w.F > 0 && scan_frames(p, s->d_x, w.x0, s->frames, w.F, G, s->d_work, s->d_pw, s->stream, &s->launches)) return JAERO_E_CUDA;
    if (w.total > w.x1)
        JB_CUDA(cudaMemcpyAsync(s->d_carry, s->d_x + (w.x1 - w.x0), (w.total - w.x1) * sizeof(double2), cudaMemcpyDeviceToDevice, s->stream));
    s->n_in = w.total; s->frames = w.f_end;
    return JAERO_OK;
}
int jaero_scan_write(jaero_scan *s, const void *iq, size_t n, int format) { return stage_iq_write(s, iq, n, format, "jaero_scan_write", jaero_scan_write_device); }
int jaero_scan_set_stream(jaero_scan *s, void *cuda_stream) { return switch_stream(s, cuda_stream); }
int jaero_scan_reset(jaero_scan *s)
{
    if (!s) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(s->device));
    JB_CUDA(cudaMemsetAsync(s->p.sum, 0, s->p.nfft * sizeof(double), s->stream));
    JB_CUDA(cudaMemsetAsync(s->p.maxh, 0, s->p.nfft * sizeof(double), s->stream));
    s->n_in = 0; s->frames = 0;
    return JAERO_OK;
}
int jaero_scan_read(jaero_scan *s, double *mean, double *max_hold, int64_t *frames)
{
    if (!s) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(s->device));
    const int N = s->p.nfft;
    if (mean) JB_CUDA(cudaMemcpyAsync(mean, s->p.sum, N * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    if (max_hold) JB_CUDA(cudaMemcpyAsync(max_hold, s->p.maxh, N * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    JB_CUDA(cudaStreamSynchronize(s->stream));
    if (mean && s->frames > 0)
        for (int i = 0; i < N; i++) mean[i] /= (double)s->frames;
    if (frames) *frames = s->frames;
    return JAERO_OK;
}

} // extern "C"

// Carrier finding (host only). The sliding order statistic of the floor: the bins are ranked once by (value, index), a Fenwick tree
// over the ranks holds the window's members, and the k-th smallest member is found by descending the tree, O(log nfft) per bin.
static void scan_floor(const double *psd, int n, int W, double q, double *floor_out)
{
    std::vector<int> order(n), rank(n), tree(n + 1, 0);
    for (int i = 0; i < n; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [psd](int a, int b) { return psd[a] < psd[b] || (psd[a] == psd[b] && a < b); });
    for (int r = 0; r < n; r++) rank[order[r]] = r;
    int top = 1;
    while (top * 2 <= n) top *= 2;
    auto add = [&](int bin, int d) { for (int j = rank[bin] + 1; j <= n; j += j & -j) tree[j] += d; };
    auto kth = [&](int k) {                                          // rank of the k-th smallest member, k from 0
        int pos = 0;
        for (int step = top; step; step >>= 1)
            if (pos + step <= n && tree[pos + step] <= k) { pos += step; k -= tree[pos]; }
        return pos;
    };
    const int k = (int)std::floor((W - 1) * q);
    for (int j = 0; j < W; j++) add(j, 1);
    int s_cur = 0;
    for (int i = 0; i < n; i++) {
        const int s = std::min(std::max(i - (W - 1) / 2, 0), n - W);
        for (; s_cur < s; s_cur++) { add(s_cur, -1); add(s_cur + W, 1); }
        floor_out[i] = psd[order[kth(k)]];
    }
}
// The floor of a spectrum of n bins over fs, once every bin is checked to be finite and >= 0: the q-quantile of a sliding window of
// window_hz (odd, 3 to n bins)
static int spectrum_floor(const double *psd, int n, double fs, double window_hz, double q, std::vector<double> &fl, const char *fn)
{
    for (int i = 0; i < n; i++)
        if (!(psd[i] >= 0) || !std::isfinite(psd[i])) return arg_error(fn, "spectrum values must be finite and >= 0");
    const double bin_hz = fs / n;
    const double x = std::min(window_hz / bin_hz, (double)n);
    const int W = std::min(std::max(2 * (int)std::floor(x / 2) + 1, 3), n);
    fl.resize(n);
    scan_floor(psd, n, W, q, fl.data());
    return JAERO_OK;
}

// Nominal half-power widths of the continuous modes.
//   OQPSK with root-raised-cosine pulses on each arm: the spectrum is a raised cosine of the symbol rate Rs = fb / 2, and a raised
//   cosine of any roll-off is at half its peak at +-Rs/2, so the half-power width is Rs: 5250 Hz at 10500 bps, 4200 Hz at 8400.
//   MSK with half-sine pulses: S(f) ~ [cos(2 pi f T) / (1 - 16 f^2 T^2)]^2 with T = 1 / fb falls to half its peak at
//   f T = 0.297241, a half-power width of 0.594482 fb: 356.7 Hz at 600 bps and 713.4 Hz at 1200.
static int scan_mode_hint(double width)
{
    static const double nominal[4] = {0.594482 * 600, 0.594482 * 1200, 4200.0, 5250.0};
    static const int modes[4] = {JAERO_MODE_MSK600, JAERO_MODE_MSK1200, JAERO_MODE_OQPSK8400, JAERO_MODE_OQPSK10500};
    if (!(width > 0)) return JAERO_MODE_UNKNOWN;
    int best = 0;
    for (int m = 1; m < 4; m++)
        if (fabs(log(width / nominal[m])) < fabs(log(width / nominal[best]))) best = m;
    const double r = width / nominal[best];
    return (r >= 0.8 && r <= 1.25) ? modes[best] : JAERO_MODE_UNKNOWN;
}

extern "C" int jaero_scan_find_carriers(const double *psd, int nfft, double input_rate, const jaero_scan_params *params,
                                        jaero_carrier *out, int cap, int *n_found)
{
    if (!psd || !n_found || (cap > 0 && !out) || cap < 0) { set_error("jaero_scan_find_carriers: bad argument"); return JAERO_E_ARG; }
    if (!pow2_nfft(nfft, 65536)) { set_error("jaero_scan_find_carriers: nfft must be a power of two from 1024 to 65536"); return JAERO_E_ARG; }
    if (!(input_rate > 0) || !std::isfinite(input_rate)) { set_error("jaero_scan_find_carriers: input_rate must be positive"); return JAERO_E_ARG; }
    const jaero_scan_params P = params ? *params : jaero_scan_params{3.0, 100e3, 0.25, 200.0, 0.0};
    if (!(P.threshold_db > 0) || !std::isfinite(P.threshold_db) || !(P.floor_window_hz > 0) || !std::isfinite(P.floor_window_hz) ||
        !(P.floor_quantile >= 0 && P.floor_quantile <= 1) || !(P.min_width_hz >= 0) || !std::isfinite(P.min_width_hz) ||
        !(P.dc_guard_hz >= 0) || !std::isfinite(P.dc_guard_hz)) {
        set_error("jaero_scan_find_carriers: parameter out of range"); return JAERO_E_ARG; }
    const int n = nfft;
    std::vector<double> fl, e(n);
    { const int r = spectrum_floor(psd, n, input_rate, P.floor_window_hz, P.floor_quantile, fl, "jaero_scan_find_carriers"); if (r) return r; }
    const double bin_hz = input_rate / n;
    for (int i = 0; i < n; i++) e[i] = psd[i] - fl[i];
    const double thr = pow(10.0, P.threshold_db / 10.0);
    auto hz = [&](double i) { return (i - n / 2) * bin_hz; };
    int found = 0;
    for (int i0 = 0; i0 < n;) {
        if (!(psd[i0] >= fl[i0] * thr)) { i0++; continue; }
        int i1 = i0;
        while (i1 + 1 < n && psd[i1 + 1] >= fl[i1 + 1] * thr) i1++;
        if ((i1 - i0 + 1) * bin_hz >= P.min_width_hz) {
            int pk = i0;
            double se = 0, sfe = 0, sf = 0, pr = 0, emax = e[i0];
            for (int i = i0; i <= i1; i++) {
                if (psd[i] > psd[pk]) pk = i;
                se += e[i]; sfe += hz(i) * e[i]; sf += fl[i];
                pr = std::max(pr, psd[i] / fl[i]);
                emax = std::max(emax, e[i]);
            }
            // The half-power level is half the mean excess over the carrier's top (its bins at or above half the largest excess),
            // not half the largest excess: the largest of many noisy bins sits well above the spectrum's true peak (+15 % for a
            // 10.5 kbps carrier averaged over 300 frames), which would narrow every width and move 10.5 kbps carriers to 8400.
            double top = 0;
            int ntop = 0;
            for (int i = i0; i <= i1; i++)
                if (e[i] >= 0.5 * emax) { top += e[i]; ntop++; }
            const double h = 0.5 * (top / ntop);
            int j = pk + 1;
            while (j < n && e[j] >= h) j++;
            const double xr = j == n ? n - 1 : (j - 1) + (e[j - 1] - h) / (e[j - 1] - e[j]);
            j = pk - 1;
            while (j >= 0 && e[j] >= h) j--;
            const double xl = j < 0 ? 0 : (j + 1) - (e[j + 1] - h) / (e[j + 1] - e[j]);
            jaero_carrier c;
            c.peak_hz = hz(pk);
            c.center_hz = se > 0 ? sfe / se : c.peak_hz;
            c.lo_hz = hz(i0); c.hi_hz = hz(i1);
            c.width_hz = (xr - xl) * bin_hz;
            c.power = se / n;
            c.snr_db = 10 * log10(se / sf);
            c.peak_db = 10 * log10(pr);
            c.floor = fl[pk];
            c.mode = scan_mode_hint(c.width_hz);
            c.flags = (fabs(c.center_hz) < P.dc_guard_hz ? JAERO_CARRIER_AT_DC : 0) | (i0 == 0 || i1 == n - 1 ? JAERO_CARRIER_AT_EDGE : 0);
            if (found < cap) out[found] = c;
            found++;
        }
        i0 = i1 + 1;
    }
    *n_found = found;
    return JAERO_OK;
}

// ------------------------------------------------------------------ mode identifier
struct jaero_ident : Stage {
    IdentPlan p;
    long long frames;                                                // complete frames per channel since create / reset (n_in: samples)
    int16_t *d_carry;                                                // [C][nfft] samples frames * hop .. n_in - 1 (fewer than nfft)
    int16_t *d_in; size_t in_cap;                                    // host writes: the PCM staged on the device, [C][n]
    int16_t *d_x; size_t x_cap;                                      // [C][carry + n] the samples the write's frames read
    double2 *d_w0, *d_w1;                                            // [G][nfft] work matrices of one pass
};

static bool ident_fs_ok(double fs) { return std::isfinite(fs) && fs >= 8000 && fs <= 192000 && fs == floor(fs); }
static int ident_pass_frames(int nfft) { return (int)std::max<long long>(1, IDENT_PASS_ELEMS / nfft); }

extern "C" {

int jaero_ident_create(double Fs, int n_channels, int nfft, int device, jaero_ident **out)
{
    const char *fn = "jaero_ident_create";
    if (!out || n_channels <= 0) { set_error(std::string(fn) + ": bad argument"); return JAERO_E_ARG; }
    if (!pow2_nfft(nfft, 16384)) { set_error(std::string(fn) + ": nfft must be a power of two from 1024 to 16384"); return JAERO_E_ARG; }
    if (!ident_fs_ok(Fs)) { set_error(std::string(fn) + ": Fs must be whole hertz from 8000 to 192000"); return JAERO_E_ARG; }
    CreateGuard<jaero_ident> guard(jaero_ident_destroy);
    { const int e = guard.begin(fn, device); if (e) return e; }
    jaero_ident *d = guard.obj;
    d->own_stream = d->stream;
    IdentPlan &p = d->p;
    p.nfft = nfft; p.hop = nfft / 2; p.n_channels = n_channels;
    const size_t work = (size_t)ident_pass_frames(nfft) * nfft;
    int rc = 0;
    rc |= owned_alloc(d, &p.sum, (size_t)n_channels * nfft);
    rc |= owned_alloc(d, &d->d_carry, (size_t)n_channels * nfft);
    rc |= owned_alloc(d, &d->d_w0, work); rc |= owned_alloc(d, &d->d_w1, work);
    if (rc) return JAERO_E_CUDA;
    double wss;
    if ((rc = four_step_tables(d, p, nfft, &wss))) return rc;
    p.inv_wss2 = 1.0 / (wss * wss);
    *out = guard.release();
    return JAERO_OK;
}
void jaero_ident_destroy(jaero_ident *d) { if (d) destroy_stage(d, {d->d_in, d->d_x}); }
int64_t jaero_ident_launch_count(const jaero_ident *d) { return d ? d->launches : 0; }

int jaero_ident_write_device(jaero_ident *d, const int16_t *d_pcm, size_t n, size_t stride)
{
    int r = pcm_write_args(d, d_pcm, n, stride, true, "jaero_ident_write_device"); if (r) return r;
    if (n == 0) return JAERO_OK;
    JB_CUDA(cudaSetDevice(d->device));
    const IdentPlan &p = d->p;
    const size_t C = (size_t)p.n_channels, B = sizeof(int16_t);
    const long long N = p.nfft;
    const FrameSpan w = frame_span(d->n_in, d->frames, N, p.hop, n);  // d_x[c][j] = sample x0 + j of channel c
    if (w.F == 0) {                                                  // no frame completes: the samples join the carry
        JB_CUDA(cudaMemcpy2DAsync(d->d_carry + w.carry, N * B, d_pcm, stride * B, n * B, C, cudaMemcpyDeviceToDevice, d->stream));
        d->n_in = w.total;
        return JAERO_OK;
    }
    const size_t pitch = (size_t)(w.carry + (long long)n);
    // every buffer is in place before anything is queued: a failed write leaves the average unchanged
    if (grow(&d->d_x, &d->x_cap, C * pitch, d->stream)) return JAERO_E_CUDA;
    if (w.carry) JB_CUDA(cudaMemcpy2DAsync(d->d_x, pitch * B, d->d_carry, N * B, w.carry * B, C, cudaMemcpyDeviceToDevice, d->stream));
    JB_CUDA(cudaMemcpy2DAsync(d->d_x + w.carry, pitch * B, d_pcm, stride * B, n * B, C, cudaMemcpyDeviceToDevice, d->stream));
    if (ident_frames(p, d->d_x, pitch, w.x0, d->frames, w.F, ident_pass_frames(p.nfft), d->d_w0, d->d_w1, d->stream, &d->launches))
        return JAERO_E_CUDA;
    if (w.total > w.x1)
        JB_CUDA(cudaMemcpy2DAsync(d->d_carry, N * B, d->d_x + (w.x1 - w.x0), pitch * B, (w.total - w.x1) * B, C, cudaMemcpyDeviceToDevice,
                                  d->stream));
    d->n_in = w.total; d->frames = w.f_end;
    return JAERO_OK;
}
int jaero_ident_write(jaero_ident *d, const int16_t *pcm, size_t n, size_t stride)
{
    return stage_pcm_write(d, pcm, n, stride, "jaero_ident_write", jaero_ident_write_device);
}
int jaero_ident_set_stream(jaero_ident *d, void *cuda_stream) { return switch_stream(d, cuda_stream); }
int jaero_ident_reset(jaero_ident *d)
{
    if (!d) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(d->device));
    JB_CUDA(cudaMemsetAsync(d->p.sum, 0, (size_t)d->p.n_channels * d->p.nfft * sizeof(double), d->stream));
    d->n_in = 0; d->frames = 0;
    return JAERO_OK;
}
int jaero_ident_read(jaero_ident *d, double *sq_mean, int64_t *frames)
{
    if (!d) { set_error("null handle"); return JAERO_E_ARG; }
    JB_CUDA(cudaSetDevice(d->device));
    const size_t total = (size_t)d->p.n_channels * d->p.nfft;
    if (sq_mean) JB_CUDA(cudaMemcpyAsync(sq_mean, d->p.sum, total * sizeof(double), cudaMemcpyDeviceToHost, d->stream));
    JB_CUDA(cudaStreamSynchronize(d->stream));
    if (sq_mean && d->frames > 0)
        for (size_t i = 0; i < total; i++) sq_mean[i] /= (double)d->frames;
    if (frames) *frames = d->frames;
    return JAERO_OK;
}

// Host only. The line pair of each JAERO rate in the squared spectrum (contract in include/jaero_b200.h).
int jaero_ident_classify(const double *sq_mean, int nfft, double Fs, const jaero_ident_params *params, jaero_ident_result *out)
{
    const char *fn = "jaero_ident_classify";
    if (!sq_mean || !out) { set_error(std::string(fn) + ": null argument"); return JAERO_E_ARG; }
    if (!pow2_nfft(nfft, 16384)) { set_error(std::string(fn) + ": nfft must be a power of two from 1024 to 16384"); return JAERO_E_ARG; }
    if (!ident_fs_ok(Fs)) { set_error(std::string(fn) + ": Fs must be whole hertz from 8000 to 192000"); return JAERO_E_ARG; }
    const jaero_ident_params P = params ? *params : jaero_ident_params{5.0, 400.0, 0.5};
    if (!std::isfinite(P.threshold_db) || !(P.floor_window_hz > 0) || !std::isfinite(P.floor_window_hz) ||
        !(P.floor_quantile >= 0 && P.floor_quantile <= 1)) { set_error(std::string(fn) + ": parameter out of range"); return JAERO_E_ARG; }
    const int n = nfft;
    std::vector<double> fl, Q(n);
    { const int e = spectrum_floor(sq_mean, n, Fs, P.floor_window_hz, P.floor_quantile, fl, fn); if (e) return e; }
    const double bin_hz = Fs / n;
    for (int i = 0; i < n; i++) Q[i] = fl[i] > 0 ? sq_mean[i] / fl[i] : 0.0;
    static const double fbs[4] = {600.0, 1200.0, 8400.0, 10500.0};
    static const int modes[4] = {JAERO_MODE_MSK600, JAERO_MODE_MSK1200, JAERO_MODE_OQPSK8400, JAERO_MODE_OQPSK10500};
    double score[4];
    long long li[4], lj[4];                                          // lower line's bin, upper line's unwrapped bin
    for (int m = 0; m < 4; m++) {
        const long long D = (long long)std::llround(fbs[m] * n / Fs);
        score[m] = -1; li[m] = lj[m] = 0;
        for (int i = 0; i < n; i++) {
            long long jmax = 0; double qmax = -1;
            for (int e = -1; e <= 1; e++) {
                const long long j = i + D + e;
                const double q = Q[(size_t)(((j % n) + n) % n)];
                if (q > qmax) { qmax = q; jmax = j; }
            }
            const double s = std::min(Q[i], qmax);
            if (s > score[m]) { score[m] = s; li[m] = i; lj[m] = jmax; }
        }
    }
    jaero_ident_result r;
    std::memset(&r, 0, sizeof r);
    int best = 0;
    for (int m = 0; m < 4; m++) {
        r.score_db[m] = score[m] > 0 ? 10 * log10(score[m]) : -HUGE_VAL;
        if (score[m] > score[best]) best = m;
    }
    double other = -HUGE_VAL;
    for (int m = 0; m < 4; m++)
        if (m != best) other = std::max(other, r.score_db[m]);
    r.margin_db = r.score_db[best] - other;
    auto refine = [&](long long k) {                                 // log-parabolic offset of the line at bin k mod n
        const int c = (int)(((k % n) + n) % n);
        const double y0 = sq_mean[(c + n - 1) % n], y1 = sq_mean[c], y2 = sq_mean[(c + 1) % n];
        if (!(y0 > 0 && y1 > 0 && y2 > 0)) return 0.0;
        const double l0 = log(y0), l1 = log(y1), l2 = log(y2), den = l0 - 2 * l1 + l2;
        if (den == 0) return 0.0;
        return std::min(0.5, std::max(-0.5, (l0 - l2) / (2 * den)));
    };
    const double di = refine(li[best]), dj = refine(lj[best]);
    const double lo = (double)li[best] + di, hi = (double)lj[best] + dj;
    r.line_hz[0] = (lo - n / 2) * bin_hz;
    r.line_hz[1] = ((double)(((lj[best] % n) + n) % n) + dj - n / 2) * bin_hz;
    r.fb_hz = (hi - lo) * bin_hz;
    const double mid = (0.5 * (lo + hi) - n / 2) * bin_hz;
    r.carrier_hz = fmod(fmod(mid, Fs) + Fs, Fs) / 2;
    r.frames = 0;
    r.mode = r.score_db[best] >= P.threshold_db ? modes[best] : JAERO_MODE_UNKNOWN;
    *out = r;
    return JAERO_OK;
}

} // extern "C"
