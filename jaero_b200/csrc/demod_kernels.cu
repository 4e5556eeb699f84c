// Single translation unit for the continuous demodulator kernels; each file also compiles on its own.
// Built with -fmad=false: see demod_device.cuh.
#include "oqpsk_demod.cu"
#include "oqpsk_pipe.cu"
#include "msk_pipe.cu"
