#include "segment_inst.cuh"
template int b200_host::segment_grid<__half>(int, int, int*);
template int b200_host::launch_segment<__half>(int, int, const ProgOp*, int, unsigned*, int, bool, unsigned long long*, cudaStream_t);
