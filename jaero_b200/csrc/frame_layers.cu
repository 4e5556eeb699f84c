// Single translation unit for the P-channel, C-channel and R/T frame layers, so that they share one copy of frame_stages.cuh
// (one scrambler table per memory space); each file also compiles on its own.
#include "pchannel.cu"
#include "cchannel.cu"
#include "rtchannel.cu"

namespace jb {

template int frame_tick<PChanState>(PChanState *, int, int *, cudaStream_t);
template int frame_tick<CChanState>(CChanState *, int, int *, cudaStream_t);
template int frame_tick<RtState>(RtState *, int, int *, cudaStream_t);
template int frame_lost<PChanState>(PChanState *, int, int, int *, cudaStream_t);
template int frame_lost<CChanState>(CChanState *, int, int, int *, cudaStream_t);
template int frame_out_reset<CChanState>(CChanState *, int, cudaStream_t);
template int frame_out_reset<RtState>(RtState *, int, cudaStream_t);

} // namespace jb
