// infidex_b200 -- CUDA translation unit of libinfidex_gpu.so (sm_90a). See include/infidex_gpu.h.
#include "ifx_api.inl"
