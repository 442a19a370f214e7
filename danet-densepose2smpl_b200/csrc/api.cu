// Error plumbing and device queries for libdanet_b200.so.
#include "common.cuh"

namespace danet {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace danet

extern "C" const char* danet_last_error(void) { return danet::g_err; }
// 3: danet_act views, danet_conv_tc_group (split-fp16 tensor-core engine); 4: one weight packer
// (danet_conv_tc_pack is stream-ordered, danet_conv_tc_pack_async is gone), danet_conv_tc_config without sub-tiles;
// 5: the network's inference launches (danet_conv2d, danet_fuse_sum, danet_maxpool3x3s2, danet_nchw_to_nhwc,
// danet_iuv_clean_global / _parts, danet_stn_params / _sample, danet_gcn_pose_head) are internal: network programs
// and danet_net_run_step are their entry
extern "C" int danet_version(void) { return 5; }
extern "C" int danet_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    DANET_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp p;
    DANET_CUDA(cudaGetDeviceProperties(&p, dev));
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    return 0;
}
