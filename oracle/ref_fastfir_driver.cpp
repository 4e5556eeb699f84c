// TEST INFRASTRUCTURE ONLY (oracle/_ref/libjaero_ref_fastfir.so).
// extern "C" wrappers around the reference's JFastFir and QJHilbertFilter (DSP.h / DSP.cpp, compiled verbatim by
// oracle/Makefile over the restated JFFT), for tests/test_fastfir_reference_cpu.py. A library of its own, so that a
// libjaero_ref.so built before these wrappers existed still loads.
#include <vector>
#include <complex>
#include "qt_shim.h"
#include "DSP.h"

extern "C" {

// JFastFir with caller taps and nfft, fed as the update() calls writes[0 .. n_writes) (sizes adding up to n)
void jref_jfastfir(const double *taps_ri, int K, int nfft, double *inout_ri, long n, const int *writes, int n_writes)
{
    JFastFir fir;
    QVector<cpx_type> k(K);
    for (int i = 0; i < K; i++) k[i] = cpx_type(taps_ri[2 * i], taps_ri[2 * i + 1]);
    fir.SetKernel(k, nfft);
    long pos = 0;
    for (int w = 0; w < n_writes && pos < n; w++) {
        QVector<cpx_type> v(writes[w]);
        for (int i = 0; i < writes[w]; i++) v[i] = cpx_type(inout_ri[2 * (pos + i)], inout_ri[2 * (pos + i) + 1]);
        fir.update(v);
        for (int i = 0; i < writes[w]; i++) { inout_ri[2 * (pos + i)] = v[i].real(); inout_ri[2 * (pos + i) + 1] = v[i].imag(); }
        pos += writes[w];
    }
}
// QJHilbertFilter's kernel as its constructor builds it (setSize(2048), DSP.cpp:754-789): 2048 complex taps
int jref_hilbert_kernel(double *out_ri)
{
    QJHilbertFilter h;
    QVector<cpx_type> k = h.getKernel();
    for (int i = 0; i < k.size(); i++) { out_ri[2 * i] = k[i].real(); out_ri[2 * i + 1] = k[i].imag(); }
    return k.size();
}

} // extern "C"
