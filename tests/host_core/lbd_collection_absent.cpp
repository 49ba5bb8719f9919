/* tests/host_core/lbd_collection_absent.cpp -- the collection calls of the C ABI (cs_lbd_collection_*) as stand-ins that refuse, so that
 * shim/binary_descriptor_matcher_b200.cpp links against the emulated build of cs_lbd.cu (lbd_host_emu.cpp), which does not emulate
 * cs_lbd_collection.cu.  The shim's pairwise forms then run on the CPU (tests/test_matcher_shim_host_emu.py); its collection forms, and pairs
 * above the pairwise calls' 16384 train codes, which go through a collection, run on the GPU only (tests/test_gpu_matcher_shim.py).  Test
 * infrastructure, never shipped. */
#include "../../include/cube_slam_b200.h"

extern "C" {
cs_lbd_collection *cs_lbd_collection_create(cs_ctx *) { return nullptr; }
void cs_lbd_collection_destroy(cs_lbd_collection *) {}
int cs_lbd_collection_add(cs_lbd_collection *, const uint8_t *, const int32_t *, int) { return CS_ERR_UNSUPPORTED; }
int cs_lbd_collection_size(const cs_lbd_collection *, int32_t *, int64_t *) { return CS_ERR_UNSUPPORTED; }
int cs_lbd_collection_match(cs_lbd_collection *, const uint8_t *, int, const uint8_t *, int, cs_dmatch *, int32_t *) { return CS_ERR_UNSUPPORTED; }
int cs_lbd_collection_knn_match(cs_lbd_collection *, const uint8_t *, int, int, const uint8_t *, int, cs_dmatch *, int32_t *) { return CS_ERR_UNSUPPORTED; }
int cs_lbd_collection_radius_match(cs_lbd_collection *, const uint8_t *, int, float, const uint8_t *, int, cs_dmatch *, int64_t, int64_t *)
{
    return CS_ERR_UNSUPPORTED;
}
}
