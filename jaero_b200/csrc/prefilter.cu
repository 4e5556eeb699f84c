// K6 — 8400 bps pre-filter: mix down -> 2049-tap RRC via streaming FFT convolution (nfft 4096) -> mix up.
//
// Replaces the `fb==8400` block at the top of OqpskDemodulator::writeData (JAERO/oqpskdemodulator.cpp:343-381). The JFastFir
// object it drives is the streaming FFT convolution of fastfir.cuh (L = nfft-K+1 = 2048), which also serves the burst
// demodulators' Hilbert filter (DSP.cpp:754-794).
//
//   pre_down_kernel        thread/channel: x[i] = mixer_fir_pre.CIS * pcm[i]        (:353-365, phases accumulated serially)
//   fir_exchange_up_kernel thread/channel: per-sample in/out exchange against the L-sample staging block (JFastFir::update)
//                                          followed by the conjugate mix-up from the saved phase (:371-379)
//   fastfir_block_kernel   CTA/channel:    overlap-save block: [history | new L] -> FFT4096 -> xH -> IFFT4096 -> last L
//                                          (fastfir.cu)
#include "demod_device.cuh"
#include "prefilter.cuh"

namespace jb {

// mix down with mixer_fir_pre (oqpskdemodulator.cpp:353-365). The oscillator itself is not advanced here: the reference
// rewinds it to the saved phase before the mix-up loop, whose end state is what persists.
__global__ void pre_down_kernel(PreParams q, const int16_t *__restrict__ pcm, size_t stride, int n)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= q.n_channels) return;
    Osc o = {q.osc[0 * q.cpad + ch], q.osc[1 * q.cpad + ch], q.osc[2 * q.cpad + ch], 0.0};
    const int16_t *row = pcm + (size_t)ch * stride;
    double2 *x = q.x + (size_t)ch * q.xstride;
    for (int i = 0; i < n; i++) {
        const double dval = ((double)row[i]) / 32768.0;
        const int t = osc_index(o.ptr);
        x[i] = make_double2(q.cos_t[t] * dval, q.sin_t[t] * dval);
        osc_next_frame(o);
    }
    // savedphase=GetPhaseDeg() (:354) ... SetPhaseDeg(savedphase) (:371): the round trip through degrees is kept
    const double saved = (360.0 * q.osc[0 * q.cpad + ch] / ((double)WTSIZE));
    Osc r = {0, 0, 0, 0};
    osc_set_phase_deg(r, saved);
    q.osc[3 * q.cpad + ch] = r.ptr;       // start pointer of the mix-up loop
}

// JFastFir::update sample exchange for samples [i0,i1) of this call + conjugate mix-up (:371-379)
__global__ void fir_exchange_up_kernel(PreParams q, FastFir f, int i0, int i1, int fill0)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= q.n_channels) return;
    double2 *x = q.x + (size_t)ch * q.xstride;
    double2 *inb = f.inblk + (size_t)ch * f.L;
    const double2 *outb = f.outblk + (size_t)ch * f.L;
    Osc o = {q.osc[3 * q.cpad + ch], q.osc[1 * q.cpad + ch], q.osc[2 * q.cpad + ch], 0.0};
    int fill = fill0;
    for (int i = i0; i < i1; i++) {
        const double2 xin = x[i];
        const double2 y = outb[fill];
        inb[fill] = xin;
        fill++;
        const int t = osc_index(o.ptr);
        x[i] = c_mul(y, make_double2(q.cos_t[t], -q.sin_t[t]));          // *= WTCISValue_conj()
        osc_next_frame(o);
    }
    q.osc[3 * q.cpad + ch] = o.ptr;
}

// end of writeData (:608): mixer_fir_pre.SetFreq(mixer2_freq_sum/i); its pointer is where the mix-up loop left it
__global__ void pre_finish_kernel(PreParams q, const double *__restrict__ m2_freq_sum, int n, double Fs)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= q.n_channels) return;
    double f = m2_freq_sum[ch] / ((double)n);
    if (f < 0) f = 0;
    q.osc[2 * q.cpad + ch] = f;
    q.osc[1 * q.cpad + ch] = (f) * ((double)WTSIZE) / Fs;
    q.osc[0 * q.cpad + ch] = q.osc[3 * q.cpad + ch];
}

int pre_down_launch(const PreParams &q, const int16_t *pcm, size_t stride, int n, cudaStream_t s)
{
    pre_down_kernel<<<(q.n_channels + 63) / 64, 64, 0, s>>>(q, pcm, stride, n);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int fir_exchange_up_launch(const PreParams &q, const FastFir &f, int i0, int i1, int fill0, cudaStream_t s)
{
    fir_exchange_up_kernel<<<(q.n_channels + 63) / 64, 64, 0, s>>>(q, f, i0, i1, fill0);
    JB_CUDA(cudaGetLastError());
    return 0;
}
int pre_finish_launch(const PreParams &q, const double *m2_freq_sum, int n, double Fs, cudaStream_t s)
{
    pre_finish_kernel<<<(q.n_channels + 63) / 64, 64, 0, s>>>(q, m2_freq_sum, n, Fs);
    JB_CUDA(cudaGetLastError());
    return 0;
}

} // namespace jb
