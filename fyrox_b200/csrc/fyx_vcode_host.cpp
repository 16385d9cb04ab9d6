// Host build of the vertex-block code (fyx_vcode.cuh) for the CPU tests: the same functions k_vcode and k_skin run.
#include "fyx_vcode.cuh"

using namespace fyx::vcode;

extern "C" {

int fyx_vcode_coded_block_bytes() { return kCodedBytes; }

// The load of one surface whose vertices are already in the raw blocks `blocks` (11 x 32 float4 each), as k_vcode does it
// (code = false: a context that keeps every block raw).  Returns the number of blocks it coded.
uint32_t fyx_vcode_load_surface(uint32_t *blocks, uint8_t *vflag, uint64_t first_vertex, uint64_t n_padded, int code)
{
    const LoadBlocks lb = load_blocks(first_vertex, n_padded);
    uint32_t coded = 0;
    for (uint64_t b = lb.first; code && b < lb.complete_end; ++b)
        if (vflag[b] == kVflagRaw && encode_block(blocks + b * kRawF4 * 4)) {
            vflag[b] = kVflagCoded;
            ++coded;
        }
    return coded;
}

// every coded block back to the raw layout, in place (k_vdecode_all)
void fyx_vcode_decode_blocks(uint32_t *blocks, uint8_t *vflag, uint64_t n_blocks)
{
    for (uint64_t b = 0; b < n_blocks; ++b) {
        if (vflag[b] != kVflagCoded) continue;
        uint32_t raw[kRawF4 * 4];
        for (int g = 0; g < kGroups; ++g) decode_group_to_raw(blocks + b * kRawF4 * 4, g, raw);
        for (int i = 0; i < kRawF4 * 4; ++i) blocks[b * kRawF4 * 4 + i] = raw[i];
        vflag[b] = kVflagRaw;
    }
}

} // extern "C"
