// fyx_vcode.cuh — the exact code of k_skin's input blocks (DESIGN.md §3): the encoder of the load, the decoder of k_skin,
// and the host build of both (fyx_vcode_host.cpp) that the CPU tests run.
//
// A raw block holds 128 vertices as 32 four-vertex groups in 11 rows of 32 float4 (x, y, z, nx, ny, nz, w0..w3, then the
// 4x u8 bone indices; fyx_internal.h): 5 632 B.  Within one block a float row spans few exponents (positions sit in a mesh's
// box, normals in [-1, 1], weights in [0, 1]).  Per row r, E_r = the largest exponent field of the row in the block; a value
// with exponent field e is stored as its sign, its 23 mantissa bits and the code k = e - E_r + 15 (1..15), and +-0 as
// k = 0 with its sign.  A block is coded only if every value of its 10 float rows is +-0 or a normal float with
// e in [E_r - 14, E_r], and E_r <= 142 (|value| < 2^16); any other block (denormals, an exponent spread over 15, large or
// non-finite values) stays raw.
//
// Decoding: the sign, k and the mantissa are the bits of the float 1.m * 2^(k - 127) (k = 0 with m = 0: +-0), which times
// 2^(E_r - 15) is the stored value.  Both factors are normal and the product is a normal float with the same mantissa, so the
// multiplication is exact: the decoded value equals the loaded one bit for bit.
//
// Coded block: the same column layout as a raw block — 10 rows of 32 float4, float4 g of a row belonging to group g — so a
// lane still reads exactly its own 10 float4, and then a 16-byte header: 5 136 B at the raw block's stride.  The 40 words
// (row-major, 4 per float4) of group g:
//   words 3r .. 3r+2  row r's 4 values, 24 bits each (k's lowest bit and the mantissa), value j at bits 24j ..
//   word 30 + p       rows 2p and 2p+1: byte j = nibble (sign << 3 | k >> 1) of row 2p's value j, row 2p+1's above it
//   words 35 .. 38    the bone-index words of the group's 4 vertices
//   word 39           0
// header: E_0..E_9 as bytes, 6 zero bytes.  Which blocks are coded is one byte per block (kVflag*).
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define FYX_VC_HD __host__ __device__ __forceinline__
#else
#define FYX_VC_HD inline
#endif

namespace fyx {
namespace vcode {

constexpr int kRows = 10;                     // float rows of a block
constexpr int kGroups = 32;                   // four-vertex groups of a block
constexpr int kRawF4 = 11 * kGroups;          // a raw block: 5 632 B (the block stride)
constexpr int kHeaderF4 = kRows * kGroups;    // float4 offset of a coded block's header
constexpr int kCodedBytes = (kHeaderF4 + 1) * 16;
constexpr int kWords = 40;                    // words of a group in a coded block
constexpr int kNibbleWord0 = 3 * kRows, kIndexWord0 = kNibbleWord0 + kRows / 2;
constexpr uint32_t kMaxE = 142;               // largest E_r whose scale 2^(E_r - 15) is a normal float

constexpr uint8_t kVflagRaw = 0, kVflagCoded = 1;

FYX_VC_HD uint32_t exp_field(const uint32_t b) { return (b >> 23) & 0xFFu; }

// value b can be coded against the row's largest exponent field E
FYX_VC_HD bool fits(const uint32_t b, const uint32_t E)
{
    if ((b << 1) == 0u) return true; // +-0
    const uint32_t e = exp_field(b);
    return e >= 1u && E <= kMaxE && e + 14u >= E; // e <= E by the choice of E
}

FYX_VC_HD uint32_t byte_perm(const uint32_t x, const uint32_t y, const uint32_t s)
{
#if defined(__CUDA_ARCH__)
    return __byte_perm(x, y, s);
#else
    const uint64_t xy = (uint64_t)y << 32 | x;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((xy >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
#endif
}

FYX_VC_HD float as_float(const uint32_t u)
{
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}

FYX_VC_HD uint32_t as_bits(const float f)
{
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
#endif
}

// one group: v[r][j] = bits of row r, vertex j; idx[j] = vertex j's bone-index word -> its 40 words (every value fits E)
FYX_VC_HD void pack_group(const uint32_t (&v)[kRows][4], const uint32_t (&idx)[4], const uint32_t (&E)[kRows], uint32_t (&w)[kWords])
{
    for (int p = kNibbleWord0; p < kWords; ++p) w[p] = 0u;
    for (int r = 0; r < kRows; ++r) {
        uint32_t L[4];
        for (int j = 0; j < 4; ++j) {
            const uint32_t b = v[r][j];
            const uint32_t k = ((b << 1) == 0u) ? 0u : exp_field(b) + 15u - E[r];
            L[j] = (k & 1u) << 23 | (b & 0x7FFFFFu);
            w[kNibbleWord0 + r / 2] |= ((b >> 31) << 3 | k >> 1) << (8 * j + 4 * (r & 1));
        }
        w[3 * r + 0] = L[0] | L[1] << 24;
        w[3 * r + 1] = L[1] >> 8 | L[2] << 16;
        w[3 * r + 2] = L[2] >> 16 | L[3] << 8;
    }
    for (int j = 0; j < 4; ++j) w[kIndexWord0 + j] = idx[j];
}

FYX_VC_HD uint32_t header_E(const uint32_t (&h)[3], const int r) { return (h[r >> 2] >> (8 * (r & 3))) & 0xFFu; }

// row r of a group: its 3 value words, its nibble word, E_r -> the 4 values
FYX_VC_HD void unpack_row(const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t nw, const int r, const uint32_t E,
                          float (&out)[4])
{
    // top byte of each value's bits: sign << 7 | k >> 1
    const uint32_t tb = (r & 1) ? ((nw & 0x80808080u) | ((nw >> 4) & 0x07070707u)) : (((nw & 0x08080808u) << 4) | (nw & 0x07070707u));
    const float scale = as_float((E + 112u) << 23); // 2^(E - 15)
    const uint32_t d[4] = {byte_perm(w0, tb, 0x4210u), byte_perm(byte_perm(w0, w1, 0x0543u), tb, 0x5210u),
                           byte_perm(byte_perm(w1, w2, 0x0432u), tb, 0x6210u), byte_perm(w2, tb, 0x7321u)};
    for (int j = 0; j < 4; ++j) {
#if defined(__CUDA_ARCH__)
        out[j] = __fmul_rn(as_float(d[j]), scale);
#else
        out[j] = as_float(d[j]) * scale;
#endif
    }
}

FYX_VC_HD void unpack_group(const uint32_t (&w)[kWords], const uint32_t (&h)[3], float (&v)[kRows][4], uint32_t (&idx)[4])
{
    for (int r = 0; r < kRows; ++r) unpack_row(w[3 * r], w[3 * r + 1], w[3 * r + 2], w[kNibbleWord0 + r / 2], r, header_E(h, r), v[r]);
    for (int j = 0; j < 4; ++j) idx[j] = w[kIndexWord0 + j];
}

// raw layout: word (r * 32 + g) * 4 + j = row r, vertex j of group g; coded: word (r * 32 + g) * 4 + c = word 4r + c of group g
FYX_VC_HD void load_raw_group(const uint32_t *raw, const int g, uint32_t (&v)[kRows][4], uint32_t (&idx)[4])
{
    for (int r = 0; r < kRows; ++r)
        for (int j = 0; j < 4; ++j) v[r][j] = raw[(r * kGroups + g) * 4 + j];
    for (int j = 0; j < 4; ++j) idx[j] = raw[(kRows * kGroups + g) * 4 + j];
}

FYX_VC_HD void store_coded_group(uint32_t *blk, const int g, const uint32_t (&w)[kWords])
{
    for (int r = 0; r < kRows; ++r)
        for (int c = 0; c < 4; ++c) blk[(r * kGroups + g) * 4 + c] = w[4 * r + c];
}

FYX_VC_HD void store_header(uint32_t *blk, const uint32_t (&E)[kRows])
{
    uint32_t *h = blk + kHeaderF4 * 4;
    h[0] = E[0] | E[1] << 8 | E[2] << 16 | E[3] << 24;
    h[1] = E[4] | E[5] << 8 | E[6] << 16 | E[7] << 24;
    h[2] = E[8] | E[9] << 8;
    h[3] = 0u;
}

// the coded block at blk back to the raw layout at raw
FYX_VC_HD void decode_group_to_raw(const uint32_t *blk, const int g, uint32_t *raw)
{
    const uint32_t h[3] = {blk[kHeaderF4 * 4], blk[kHeaderF4 * 4 + 1], blk[kHeaderF4 * 4 + 2]};
    uint32_t w[kWords], idx[4];
    float v[kRows][4];
    for (int r = 0; r < kRows; ++r)
        for (int c = 0; c < 4; ++c) w[4 * r + c] = blk[(r * kGroups + g) * 4 + c];
    unpack_group(w, h, v, idx);
    for (int r = 0; r < kRows; ++r)
        for (int j = 0; j < 4; ++j) raw[(r * kGroups + g) * 4 + j] = as_bits(v[r][j]);
    for (int j = 0; j < 4; ++j) raw[(kRows * kGroups + g) * 4 + j] = idx[j];
}

// The blocks a surface's load writes: its vertices [first_vertex, first_vertex + n_padded) touch blocks [first, touched_end)
// and complete [first, complete_end); the last one may wait for the next surface's vertices.  A block is coded once, when
// it is complete: no later surface writes into it again.
struct LoadBlocks {
    uint64_t first, complete_end, touched_end;
};
FYX_VC_HD LoadBlocks load_blocks(const uint64_t first_vertex, const uint64_t n_padded)
{
    return LoadBlocks{first_vertex >> 7, (first_vertex + n_padded) >> 7, (first_vertex + n_padded + 127) >> 7};
}

// host: code the raw block in place; false (block untouched) when it must stay raw
inline bool encode_block(uint32_t *blk)
{
    uint32_t E[kRows] = {};
    for (int g = 0; g < kGroups; ++g)
        for (int r = 0; r < kRows; ++r)
            for (int j = 0; j < 4; ++j) {
                const uint32_t e = exp_field(blk[(r * kGroups + g) * 4 + j]);
                if (e > E[r]) E[r] = e;
            }
    for (int g = 0; g < kGroups; ++g)
        for (int r = 0; r < kRows; ++r)
            for (int j = 0; j < 4; ++j)
                if (!fits(blk[(r * kGroups + g) * 4 + j], E[r])) return false;
    static uint32_t w[kGroups][kWords]; // host tests only
    for (int g = 0; g < kGroups; ++g) {
        uint32_t v[kRows][4], idx[4];
        load_raw_group(blk, g, v, idx);
        pack_group(v, idx, E, w[g]);
    }
    for (int g = 0; g < kGroups; ++g) store_coded_group(blk, g, w[g]);
    store_header(blk, E);
    return true;
}

#if defined(__CUDACC__)
// device: one warp codes the raw block at `blk` in place (lane = group); returns whether it did (warp-uniform)
__device__ __forceinline__ bool encode_block_warp(uint32_t *blk, const uint32_t lane)
{
    uint32_t v[kRows][4], idx[4], E[kRows];
    load_raw_group(blk, (int)lane, v, idx);
    bool ok = true;
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
        uint32_t m = 0u;
#pragma unroll
        for (int j = 0; j < 4; ++j) m = max(m, exp_field(v[r][j]));
        E[r] = __reduce_max_sync(0xFFFFFFFFu, m);
#pragma unroll
        for (int j = 0; j < 4; ++j) ok &= fits(v[r][j], E[r]);
    }
    if (!__all_sync(0xFFFFFFFFu, ok)) return false;
    uint32_t w[kWords];
    pack_group(v, idx, E, w);
    __syncwarp(); // every lane holds its raw group before the coded block overwrites it
    store_coded_group(blk, (int)lane, w);
    if (lane == 0) store_header(blk, E);
    return true;
}
#endif

} // namespace vcode
} // namespace fyx
