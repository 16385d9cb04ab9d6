// fyx_drawprep.cu — N3 (SURVEY §8f): the step right after the cull.
//
// The reference, for every node the DFS of RenderDataBundleStorage::from_graph accepts, runs
// Mesh::collect_render_data (scene/mesh/mod.rs:691-805): sort index of the node's global position
// (RenderContext::calculate_sorting_index, renderer/bundle.rs:118-127), then one push() per surface into the
// bundle keyed by (material, surface data, render path) (bundle.rs:1248-1278); RenderDataBundle::write_uniforms
// later writes `world` and `view_projection * world` per instance (bundle.rs:483-487).  Here the visible list of
// one frustum becomes, in three launches, instance arrays grouped by bundle (a counting sort keyed by the
// host-assigned bundle id) plus the bundle table (first, count, sort index of the first-pushed instance).
// HBM-bound gather/scatter: per instance 4+4 B of list + 48 B G + 4 B flags read, 128+8+4 B written.
#include "fyx_internal.h"

namespace fyx {

namespace {

// RenderContext::calculate_sorting_index: z of view_matrix.transform_point(global_position) (nalgebra: divided
// by n = row3·p + m33 unless n == 0), * 1000, `as i64` (saturating, NaN -> 0), u64::MAX/2 saturating_add_signed.
__device__ __forceinline__ uint64_t sorting_index(const float *view, const float px, const float py, const float pz)
{
    const float n = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(view[3], px), FYX_MUL(view[7], py)), FYX_MUL(view[11], pz)), view[15]);
    float z = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(view[2], px), FYX_MUL(view[6], py)), FYX_MUL(view[10], pz)), view[14]);
    if (n != 0.0f) z = __fdiv_rn(z, n);
    const float zf = FYX_MUL(z, 1000.0f);
    const long long d = __float2ll_rz(zf); // cvt.rzi.s64.f32: saturates, NaN -> 0, like Rust's `as i64`
    const uint64_t center = 0xFFFFFFFFFFFFFFFFull / 2ull;
    if (d >= 0) {
        const uint64_t ud = (uint64_t)d;
        return (center > 0xFFFFFFFFFFFFFFFFull - ud) ? 0xFFFFFFFFFFFFFFFFull : center + ud;
    }
    const uint64_t ud = (uint64_t)(-(d + 1)) + 1ull;
    return (ud > center) ? 0ull : center - ud;
}

// surfaces of the visible entry's node: (first, count) — count 0 = the default single surface
__device__ __forceinline__ uint2 surfaces_of(const InstParams &ip, const uint32_t slot)
{
    return ip.ms_range ? ip.ms_range[slot] : make_uint2(0u, 0u);
}
__device__ __forceinline__ uint32_t warp_max_u32(const uint32_t v) { return __reduce_max_sync(0xFFFFFFFFu, v); }

// the node's dense dynamic index (FYX_NONE = no surface of it is batched)
__device__ __forceinline__ uint32_t dyn_node(const InstParams &ip, const uint32_t slot) { return ip.dyn_of_slot ? ip.dyn_of_slot[slot] : FYX_NONE; }
// surface k of dynamic node d is batched, not pushed (scene/mesh/mod.rs:739-753)
__device__ __forceinline__ bool dyn_surface(const InstParams &ip, const uint32_t d, const uint32_t k)
{
    if (d == FYX_NONE) return false;
    for (uint32_t j = ip.dyn_item_first[d]; j < ip.dyn_item_first[d + 1]; ++j)
        if (ip.dyn_ordinal[j] == k || ip.dyn_ordinal[j] == FYX_NONE) return true;
    return false;
}

// the segment (shadow map of the group) that owns list position i: the last map whose first entry is <= the entry (maps with
// an empty list share their first with the next map and lose to it)
__device__ __forceinline__ uint32_t segment_of(const InstParams &ip, const uint32_t i)
{
    const uint32_t e = ip.maps[ip.map0].first + i;
    uint32_t lo = 0u, hi = ip.n_seg - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (ip.maps[ip.map0 + mid].first <= e) lo = mid;
        else hi = mid - 1u;
    }
    return lo;
}

// pass 1: sort index per visible entry, bundle histogram over its surfaces (Mesh::collect_render_data pushes one instance per
// surface, all with the node's sort index, scene/mesh/mod.rs:726-805), first-pushed instance per bundle.  kSeg: the list is
// several shadow maps; each entry takes its map's view matrix and counts into its map's bins.
template <bool kSeg> __device__ __forceinline__ void inst_keys(const NodeArrays &a, const InstParams &ip)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    const bool valid = i < ip.n;
    uint32_t slot = 0u, nsurf = 0u, ninst = 0u, seg = FYX_NONE, bin0 = 0u, dn = FYX_NONE;
    uint2 sr = make_uint2(0u, 0u);
    unsigned long long key = ~0ull;
    if (valid) {
        slot = ip.vis_slot[i];
        // Base::global_position() = translation column of the global transform
        const float px = a.G[0][slot].w, py = a.G[1][slot].w, pz = a.G[2][slot].w;
        if constexpr (kSeg) {
            seg = segment_of(ip, i);
            bin0 = seg * ip.n_bundle_ids;
            ip.tmp_sort[i] = sorting_index(ip.views + (size_t)(ip.map0 + seg) * 16u, px, py, pz);
        } else {
            ip.tmp_sort[i] = sorting_index(ip.view, px, py, pz);
        }
        const uint32_t rank = ip.rank_of_slot ? ip.rank_of_slot[slot] : ip.vis_node[i];
        key = ((unsigned long long)rank << 32) | i;
        sr = surfaces_of(ip, slot);
        nsurf = ninst = sr.y ? sr.y : 1u;
        dn = dyn_node(ip, slot);
        if (dn != FYX_NONE)
            for (uint32_t k = 0; k < nsurf; ++k) ninst -= dyn_surface(ip, dn, k) ? 1u : 0u;
    }
    const int lane = threadIdx.x & 31;
    if constexpr (kSeg) { // instances per map (a map's entries are contiguous: one or two atomics per warp)
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, seg);
        const uint32_t sum = __reduce_add_sync(peers, ninst);
        if (valid && lane == __ffs(peers) - 1) atomicAdd(ip.seg_inst + seg, sum);
    }
    const uint32_t rounds = warp_max_u32(nsurf);
    for (uint32_t k = 0; k < rounds; ++k) {
        const bool act = k < nsurf && !dyn_surface(ip, dn, k);
        uint32_t b = 0xFFFFFFFFu;
        if (act) b = bin0 + (sr.y ? ip.ms_bundle[sr.x + k] : (ip.bundle_of_slot ? ip.bundle_of_slot[slot] : 0u));
        // warp-aggregated histogram: one atomic per distinct bin in the warp
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, b);
        if (act) {
            if ((peers & ((1u << lane) - 1u)) == 0u) atomicAdd(ip.hist + b, (uint32_t)__popc(peers));
            // the minimum only ever decreases: a plain read is a safe filter in front of the atomic
            if (key < *reinterpret_cast<volatile unsigned long long *>(ip.first_key + b)) atomicMin(ip.first_key + b, key);
        }
    }
}

__global__ void __launch_bounds__(kBlock) k_inst_keys(const NodeArrays a, const InstParams ip) { inst_keys<false>(a, ip); }
__global__ void __launch_bounds__(kBlock) k_shadow_inst_keys(const NodeArrays a, const InstParams ip) { inst_keys<true>(a, ip); }

// pass 2 (one CTA): exclusive scan of the histogram -> first instance of every bundle, table of the non-empty
// bundles; the histogram is zeroed again (pass 3 uses it as the scatter cursor)
constexpr int kScanBlock = 1024;
__global__ void __launch_bounds__(kScanBlock) k_inst_scan(const InstParams ip)
{
    __shared__ uint32_t s_wsum[2][kScanBlock / 32];
    __shared__ uint32_t s_carry[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry[0] = s_carry[1] = 0u;
    __syncthreads();
    for (uint32_t base = 0; base < ip.n_bundle_ids; base += kScanBlock) {
        const uint32_t b = base + threadIdx.x;
        const uint32_t c = (b < ip.n_bundle_ids) ? ip.hist[b] : 0u;
        const uint32_t ne = c ? 1u : 0u;
        uint32_t xc = c, xn = ne; // inclusive warp scans
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t tc = __shfl_up_sync(0xFFFFFFFFu, xc, d), tn = __shfl_up_sync(0xFFFFFFFFu, xn, d);
            if (lane >= d) { xc += tc; xn += tn; }
        }
        if (lane == 31) { s_wsum[0][warp] = xc; s_wsum[1][warp] = xn; }
        __syncthreads();
        if (warp == 0) {
            uint32_t wc = s_wsum[0][lane], wn = s_wsum[1][lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t tc = __shfl_up_sync(0xFFFFFFFFu, wc, d), tn = __shfl_up_sync(0xFFFFFFFFu, wn, d);
                if (lane >= d) { wc += tc; wn += tn; }
            }
            s_wsum[0][lane] = wc; // inclusive over warps
            s_wsum[1][lane] = wn;
        }
        __syncthreads();
        const uint32_t off = s_carry[0] + (warp ? s_wsum[0][warp - 1] : 0u) + xc - c;
        const uint32_t k = s_carry[1] + (warp ? s_wsum[1][warp - 1] : 0u) + xn - ne;
        if (b < ip.n_bundle_ids) {
            ip.offset[b] = off;
            ip.hist[b] = 0u;
            if (c) {
                fyx_bundle r;
                r.id = b;
                r.first = off;
                r.count = c;
                r.reserved = 0u;
                r.sort_index = ip.tmp_sort[(uint32_t)(ip.first_key[b] & 0xFFFFFFFFull)];
                ip.o_bundles[k] = r;
            }
        }
        __syncthreads();
        if (threadIdx.x == kScanBlock - 1) {
            s_carry[0] += s_wsum[0][kScanBlock / 32 - 1];
            s_carry[1] += s_wsum[1][kScanBlock / 32 - 1];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        ip.o_totals[0] = s_carry[1];
        ip.o_totals[1] = s_carry[0]; // instances = sum of the histogram
    }
}

// Device-wide exclusive scan of the (segment, bundle) bins of a shadow group, in three launches: per-tile sums, one CTA
// that scans the tile sums and the segments' instance counts, and a downsweep that writes every bin's first instance,
// the compacted bundle table in (segment, id) order and each segment's first bundle.  kScanTile bins per CTA of 1024
// threads, four consecutive bins per thread.
constexpr int kBinThreads = 1024;
static_assert(kScanTile == 4u * kBinThreads, "four bins per thread");

// (instances, bundles) of a thread's four bins, summed over the CTA; every thread gets the CTA-wide exclusive prefix of its
// own pair and the CTA total
__device__ __forceinline__ uint2 cta_exclusive_scan(const uint2 v, uint2 &total)
{
    __shared__ uint2 s_w[kBinThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint2 x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t tx = __shfl_up_sync(0xFFFFFFFFu, x.x, d), ty = __shfl_up_sync(0xFFFFFFFFu, x.y, d);
        if (lane >= d) { x.x += tx; x.y += ty; }
    }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint2 w = s_w[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t tx = __shfl_up_sync(0xFFFFFFFFu, w.x, d), ty = __shfl_up_sync(0xFFFFFFFFu, w.y, d);
            if (lane >= d) { w.x += tx; w.y += ty; }
        }
        s_w[lane] = w; // inclusive over warps
    }
    __syncthreads();
    total = s_w[kBinThreads / 32 - 1];
    const uint2 before = warp ? s_w[warp - 1] : make_uint2(0u, 0u);
    const uint2 r = make_uint2(before.x + x.x - v.x, before.y + x.y - v.y);
    __syncthreads(); // s_w is reused by the next call
    return r;
}

__device__ __forceinline__ uint4 load_bins(const InstParams &ip, const uint32_t bin0, const uint32_t n_bins)
{
    uint4 c = make_uint4(0u, 0u, 0u, 0u);
    if (bin0 + 3u < n_bins) return *reinterpret_cast<const uint4 *>(ip.hist + bin0); // 16-B aligned: bin0 % 4 == 0
    if (bin0 < n_bins) c.x = ip.hist[bin0];
    if (bin0 + 1u < n_bins) c.y = ip.hist[bin0 + 1u];
    if (bin0 + 2u < n_bins) c.z = ip.hist[bin0 + 2u];
    return c;
}

__global__ void __launch_bounds__(kBinThreads) k_bin_reduce(const InstParams ip)
{
    pdl_trigger();
    pdl_wait(); // the histogram of the keys pass
    const uint32_t n_bins = ip.n_seg * ip.n_bundle_ids;
    const uint4 c = load_bins(ip, blockIdx.x * kScanTile + threadIdx.x * 4u, n_bins);
    const uint2 v = make_uint2(c.x + c.y + c.z + c.w, (c.x != 0u) + (c.y != 0u) + (c.z != 0u) + (c.w != 0u));
    uint2 total;
    cta_exclusive_scan(v, total);
    if (threadIdx.x == 0) ip.tile_sum[blockIdx.x] = total;
}

// one CTA: tile sums -> their exclusive prefix (in place), segment instance counts -> every segment's first instance, totals
__global__ void __launch_bounds__(kBinThreads) k_bin_scan(const InstParams ip, const uint32_t n_tiles)
{
    __shared__ uint2 s_carry;
    pdl_trigger();
    pdl_wait(); // the tile sums
    if (threadIdx.x == 0) s_carry = make_uint2(0u, 0u);
    __syncthreads();
    for (uint32_t base = 0; base < n_tiles; base += kBinThreads) {
        const uint32_t t = base + threadIdx.x;
        const uint2 v = t < n_tiles ? ip.tile_sum[t] : make_uint2(0u, 0u);
        uint2 total;
        const uint2 ex = cta_exclusive_scan(v, total);
        if (t < n_tiles) ip.tile_sum[t] = make_uint2(s_carry.x + ex.x, s_carry.y + ex.y);
        __syncthreads();
        if (threadIdx.x == 0) s_carry = make_uint2(s_carry.x + total.x, s_carry.y + total.y);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        ip.o_totals[0] = s_carry.y;
        ip.o_totals[1] = s_carry.x;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry = make_uint2(0u, 0u);
    __syncthreads();
    for (uint32_t base = 0; base < ip.n_seg; base += kBinThreads) {
        const uint32_t sg = base + threadIdx.x;
        const uint2 v = make_uint2(sg < ip.n_seg ? ip.seg_inst[sg] : 0u, 0u);
        uint2 total;
        const uint2 ex = cta_exclusive_scan(v, total);
        if (sg < ip.n_seg) ip.seg_first[sg] = ip.base_inst + s_carry.x + ex.x;
        __syncthreads();
        if (threadIdx.x == 0) s_carry.x += total.x;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kBinThreads) k_bin_downsweep(const InstParams ip)
{
    pdl_trigger();
    pdl_wait(); // the tile prefixes and the segments' first instances
    const uint32_t n_bins = ip.n_seg * ip.n_bundle_ids;
    const uint32_t bin0 = blockIdx.x * kScanTile + threadIdx.x * 4u;
    const uint4 c4 = load_bins(ip, bin0, n_bins);
    const uint32_t c[4] = {c4.x, c4.y, c4.z, c4.w};
    const uint2 v = make_uint2(c[0] + c[1] + c[2] + c[3], (c[0] != 0u) + (c[1] != 0u) + (c[2] != 0u) + (c[3] != 0u));
    uint2 total;
    const uint2 ex = cta_exclusive_scan(v, total);
    const uint2 tb = ip.tile_sum[blockIdx.x];
    uint32_t off = ip.base_inst + tb.x + ex.x, k = ip.base_bundle + tb.y + ex.y;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t bin = bin0 + j;
        if (bin >= n_bins) break;
        const uint32_t seg = bin / ip.n_bundle_ids, id = bin - seg * ip.n_bundle_ids;
        if (id == 0u) ip.seg_bfirst[seg] = k;
        ip.offset[bin] = off;
        ip.hist[bin] = 0u; // the scatter cursor
        if (c[j]) {
            fyx_bundle r;
            r.id = id;
            r.first = off - ip.seg_first[seg]; // relative to the map's instances
            r.count = c[j];
            r.reserved = 0u;
            r.sort_index = ip.tmp_sort[(uint32_t)(ip.first_key[bin] & 0xFFFFFFFFull)];
            ip.o_bundles[k] = r;
            ++k;
        }
        off += c[j];
    }
}

// pass 3: scatter into bundle order; matrices are written by 8 lanes per instance (one float4 column each), so a
// warp store covers four whole 128-byte instance records.  kSeg: the bins and view_projection of each entry's map.
template <bool kSeg> __device__ __forceinline__ void inst_scatter(const NodeArrays &a, const InstParams &ip)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool valid = i < ip.n;
    uint32_t slot = 0u, nsurf = 0u, node_flags = 0u, bin0 = 0u, map = 0u, dn = FYX_NONE;
    uint2 sr = make_uint2(0u, 0u);
    if (valid) {
        slot = ip.vis_slot[i];
        sr = surfaces_of(ip, slot);
        nsurf = sr.y ? sr.y : 1u;
        dn = dyn_node(ip, slot);
        node_flags = a.flags[slot];
        if constexpr (kSeg) {
            const uint32_t seg = segment_of(ip, i);
            bin0 = seg * ip.n_bundle_ids;
            map = ip.map0 + seg;
        }
    }
    const uint32_t rounds = warp_max_u32(nsurf);
    for (uint32_t k = 0; k < rounds; ++k) {
        const bool act = k < nsurf && !dyn_surface(ip, dn, k);
        uint32_t b = 0xFFFFFFFFu, pos = 0u, skin = FYX_NONE;
        if (act) {
            b = bin0 + (sr.y ? ip.ms_bundle[sr.x + k] : (ip.bundle_of_slot ? ip.bundle_of_slot[slot] : 0u));
            skin = sr.y ? ip.ms_skin[sr.x + k] : ip.surf_of_slot[slot];
        }
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, b);
        uint32_t base = 0u;
        const int leader = __ffs(peers) - 1;
        if (act && lane == leader) base = ip.offset[b] + atomicAdd(ip.hist + b, (uint32_t)__popc(peers));
        base = __shfl_sync(0xFFFFFFFFu, base, leader);
        if (act) {
            pos = base + __popc(peers & ((1u << lane) - 1u));
            ip.o_node[pos] = ip.vis_node[i];
            ip.o_sort[pos] = ip.tmp_sort[i];
            ip.o_surf[pos] = k;
            ip.o_skin[pos] = skin;
        }
        // the instance's world matrix: identity for a skinned surface (its vertices are placed by the bone palette,
        // scene/mesh/mod.rs:733-737) and for a static batch (:716), else the node's global transform
        const bool ident = act && ((skin != FYX_NONE) || (node_flags & FYX_NODE_STATIC_BATCH));
        const int j = lane & 7, c = j & 3;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int e = q * 4 + (lane >> 3);
            const uint32_t pe = __shfl_sync(0xFFFFFFFFu, pos, e);
            const uint32_t se = __shfl_sync(0xFFFFFFFFu, slot, e);
            const bool ve = __shfl_sync(0xFFFFFFFFu, (int)act, e) != 0;
            const bool ie = __shfl_sync(0xFFFFFFFFu, (int)ident, e) != 0;
            uint32_t me = 0u;
            if constexpr (kSeg) me = __shfl_sync(0xFFFFFFFFu, map, e);
            if (!ve) continue;
            float w0, w1, w2, w3 = (c == 3) ? 1.0f : 0.0f;
            if (ie) {
                w0 = (c == 0) ? 1.0f : 0.0f;
                w1 = (c == 1) ? 1.0f : 0.0f;
                w2 = (c == 2) ? 1.0f : 0.0f;
            } else {
                const float4 r0 = a.G[0][se], r1 = a.G[1][se], r2 = a.G[2][se];
                w0 = (c == 0) ? r0.x : (c == 1) ? r0.y : (c == 2) ? r0.z : r0.w;
                w1 = (c == 0) ? r1.x : (c == 1) ? r1.y : (c == 2) ? r1.z : r1.w;
                w2 = (c == 0) ? r2.x : (c == 1) ? r2.y : (c == 2) ? r2.z : r2.w;
            }
            float4 o;
            if (j < 4) {
                o = make_float4(w0, w1, w2, w3);
            } else {
                // (view_projection * world)[r, c], nalgebra order (Appendix A1), full 4x4: VP is projective
                const float *m;
                if constexpr (kSeg) m = ip.maps[me].view_projection;
                else m = ip.vp;
                o.x = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(m[0], w0), FYX_MUL(m[4], w1)), FYX_MUL(m[8], w2)), FYX_MUL(m[12], w3));
                o.y = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(m[1], w0), FYX_MUL(m[5], w1)), FYX_MUL(m[9], w2)), FYX_MUL(m[13], w3));
                o.z = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(m[2], w0), FYX_MUL(m[6], w1)), FYX_MUL(m[10], w2)), FYX_MUL(m[14], w3));
                o.w = FYX_ADD(FYX_ADD(FYX_ADD(FYX_MUL(m[3], w0), FYX_MUL(m[7], w1)), FYX_MUL(m[11], w2)), FYX_MUL(m[15], w3));
            }
            ip.o_mats[(size_t)pe * 8u + j] = o;
        }
    }
}

__global__ void __launch_bounds__(kBlock) k_inst_scatter(const NodeArrays a, const InstParams ip) { inst_scatter<false>(a, ip); }
__global__ void __launch_bounds__(kBlock) k_shadow_inst_scatter(const NodeArrays a, const InstParams ip) { inst_scatter<true>(a, ip); }

// ---- Dynamic batching: one pack's dynamic pass (DynParams) ----
// the segment of list entry i: the last whose first entry is <= i (an empty segment shares its first with the next and loses)
__device__ __forceinline__ uint32_t dyn_segment(const DynParams &dp, const uint32_t i)
{
    uint32_t lo = 0u, hi = dp.n_seg - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (dp.seg_first[mid] <= i) lo = mid;
        else hi = mid - 1u;
    }
    return lo;
}

// mark: the segment's dynamic nodes as bits (dense index = push order), its items, vertices and triangles per layout; the
// counts are summed over the warp's lanes that hit the same (segment, layout) before one atomic per counter.  A quad node
// pushes nothing in a shadow pass, and a sprite nothing without cast_shadows (sprite.rs:327-329, rectangle.rs:328-330).
__global__ void __launch_bounds__(kBlock) k_dyn_mark(const NodeArrays a, const DynParams dp)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    uint32_t d = FYX_NONE, seg = 0u, j0 = 0u, nj = 0u;
    if (i < dp.n) {
        const uint32_t slot = dp.vis_slot[i];
        d = dp.dyn_of_slot[slot];
        if (d != FYX_NONE) {
            const uint32_t kind = dp.items[dp.item_first[d]].kind;
            if (kind != kDynMesh && (dp.shadow || (kind == FYX_SPRITE_3D && !(a.flags[slot] & FYX_NODE_CAST_SHADOWS)))) d = FYX_NONE;
        }
    }
    if (d != FYX_NONE) {
        seg = dyn_segment(dp, i);
        atomicOr(dp.bitmap + (size_t)seg * dp.words + (d >> 5), 1u << (d & 31u));
        j0 = dp.item_first[d];
        nj = dp.item_first[d + 1] - j0;
    }
    const uint32_t rounds = warp_max_u32(nj);
    const int lane = threadIdx.x & 31;
    for (uint32_t k = 0; k < rounds; ++k) {
        uint32_t key = FYX_NONE, nv = 0u, nt = 0u;
        if (k < nj) {
            const DynItemDev it = dp.items[j0 + k];
            key = seg * dp.n_layouts + it.layout;
            nv = it.n_verts;
            nt = it.n_tris;
        }
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key);
        const uint32_t cnt = __popc(peers), sv = __reduce_add_sync(peers, nv), st = __reduce_add_sync(peers, nt);
        if (key != FYX_NONE && lane == __ffs(peers) - 1) {
            uint32_t *c = dp.counts + (size_t)key * 3u;
            atomicAdd(c, cnt);
            atomicAdd(c + 1, sv);
            atomicAdd(c + 2, st);
        }
    }
}

constexpr unsigned long long kDynEmpty = ~0ull; // never a sort index (those stop at u64::MAX - 1) nor a bundle key (batch key < 2^24)
__device__ __forceinline__ uint32_t dyn_hash(unsigned long long k, const uint32_t mask)
{
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (uint32_t)k & mask;
}
// the smallest value inserted with key k wins
__device__ __forceinline__ void dyn_insert(unsigned long long *keys, uint32_t *vals, const uint32_t mask, const unsigned long long k, const uint32_t v)
{
    for (uint32_t h = dyn_hash(k, mask);; h = (h + 1u) & mask) {
        const unsigned long long prev = atomicCAS(keys + h, kDynEmpty, k);
        if (prev == kDynEmpty || prev == k) {
            atomicMin(vals + h, v);
            return;
        }
    }
}
__device__ __forceinline__ uint32_t dyn_lookup(const unsigned long long *keys, const uint32_t *vals, const uint32_t mask, const unsigned long long k)
{
    for (uint32_t h = dyn_hash(k, mask);; h = (h + 1u) & mask)
        if (__ldcg(keys + h) == k) return __ldcg(vals + h);
}

// One CTA per segment, in the reference's push order (items at seg_item0[seg] + p, p = push position):
//   1. the items of the marked nodes, node after node (bitmap order = DFS rank order);
//   2. each item's first vertex and triangle in its layout's stream (a scan per layout the segment uses);
//   3. the bundle key (batch key, sort index): equal sort indices are named by their first item (hash 1), equal keys by their
//      first item (hash 2) — the bundle's first push;
//   4. runs (an item starts an instance unless the previous item went to the same bundle: last_bundle_id) and bundles, both
//      numbered in push order;
//   5. instances per bundle, their scan, and each run's place in its bundle (push order within the bundle).
__global__ void __launch_bounds__(kBinThreads) k_dyn_order(const NodeArrays a, const DynParams dp)
{
    __shared__ uint32_t s_b[kBinThreads];
    const uint32_t seg = blockIdx.x, t = threadIdx.x;
    const uint32_t i0 = dp.seg_item0[seg], ni = dp.seg_item0[seg + 1] - i0;
    if (ni == 0u) {
        if (t == 0) dp.o_seg[seg * 2] = dp.o_seg[seg * 2 + 1] = 0u;
        return;
    }
    const uint32_t hmask = dp.seg_hmask[seg];
    unsigned long long *hk1 = dp.hkey + dp.seg_hash0[seg], *hk2 = hk1 + hmask + 1u;
    uint32_t *hv1 = dp.hval + dp.seg_hash0[seg], *hv2 = hv1 + hmask + 1u;
    // Every thread keeps the running carries in registers: the scan's totals are the same in every thread, so no thread
    // writes a shared carry that another may still be reading.
    uint2 total, carry = make_uint2(0u, 0u);
    // 1. items in push order
    for (uint32_t w0 = 0; w0 < dp.words; w0 += kBinThreads) {
        const uint32_t w = w0 + t;
        const uint32_t bits = w < dp.words ? dp.bitmap[(size_t)seg * dp.words + w] : 0u;
        uint32_t cnt = 0u;
        for (uint32_t b = bits; b; b &= b - 1u) {
            const uint32_t d = w * 32u + (__ffs(b) - 1);
            cnt += dp.item_first[d + 1] - dp.item_first[d];
        }
        uint32_t pos = carry.x + cta_exclusive_scan(make_uint2(cnt, 0u), total).x;
        for (uint32_t b = bits; b; b &= b - 1u) {
            const uint32_t d = w * 32u + (__ffs(b) - 1);
            for (uint32_t j = dp.item_first[d]; j < dp.item_first[d + 1]; ++j) dp.ord_item[i0 + pos++] = j;
        }
        carry.x += total.x;
    }
    __syncthreads(); // the items
    // 2. vertex and triangle offsets in each layout's stream
    for (uint32_t l = 0; l < dp.n_layouts; ++l) {
        if (dp.counts[((size_t)seg * dp.n_layouts + l) * 3u] == 0u) continue;
        carry = make_uint2(0u, 0u);
        for (uint32_t p0 = 0; p0 < ni; p0 += kBinThreads) {
            const uint32_t p = p0 + t;
            uint2 v = make_uint2(0u, 0u);
            if (p < ni) {
                const DynItemDev it = dp.items[dp.ord_item[i0 + p]];
                if (it.layout == l) v = make_uint2(it.n_verts, it.n_tris);
            }
            const uint2 ex = cta_exclusive_scan(v, total);
            if (p < ni && dp.items[dp.ord_item[i0 + p]].layout == l) {
                dp.voff[i0 + p] = carry.x + ex.x;
                dp.toff[i0 + p] = carry.y + ex.y;
            }
            carry = make_uint2(carry.x + total.x, carry.y + total.y);
        }
    }
    __syncthreads(); // the offsets
    // 3. the bundle keys
    const float *view = dp.views + (size_t)seg * 16u;
    for (uint32_t p = t; p < ni; p += kBinThreads) {
        const uint32_t slot = dp.items[dp.ord_item[i0 + p]].slot;
        const uint64_t si = sorting_index(view, a.G[0][slot].w, a.G[1][slot].w, a.G[2][slot].w);
        dp.sidx[i0 + p] = si;
        dyn_insert(hk1, hv1, hmask, si, p);
    }
    __syncthreads();
    for (uint32_t p = t; p < ni; p += kBinThreads) {
        const uint64_t k2 = ((uint64_t)dp.items[dp.ord_item[i0 + p]].batch_key << 32) | dyn_lookup(hk1, hv1, hmask, dp.sidx[i0 + p]);
        dp.key2[i0 + p] = k2;
        dyn_insert(hk2, hv2, hmask, k2, p);
    }
    __syncthreads();
    // 4. runs and bundles in push order
    carry = make_uint2(0u, 0u);
    for (uint32_t p0 = 0; p0 < ni; p0 += kBinThreads) {
        const uint32_t p = p0 + t;
        uint32_t bfirst = FYX_NONE, run_start = 0u, bstart = 0u;
        uint64_t k2 = 0;
        if (p < ni) {
            k2 = __ldcg(dp.key2 + i0 + p);
            bfirst = dyn_lookup(hk2, hv2, hmask, k2);
            run_start = (p == 0u || __ldcg(dp.key2 + i0 + p - 1u) != k2) ? 1u : 0u;
            bstart = bfirst == p ? 1u : 0u;
        }
        const uint2 ex = cta_exclusive_scan(make_uint2(run_start, bstart), total);
        const uint32_t r = carry.x + ex.x + run_start - 1u; // the item's run
        if (p < ni) {
            dp.run_of[i0 + p] = r;
            if (bstart) {
                const uint32_t b = carry.y + ex.y;
                dp.bord[i0 + p] = b;
                const DynItemDev it = dp.items[dp.ord_item[i0 + p]];
                fyx_dynamic_bundle rec;
                rec.batch_key = it.batch_key;
                rec.layout_id = it.layout;
                rec.first = rec.count = 0u;
                rec.sort_index = dp.sidx[i0 + p];
                dp.o_bundles[i0 + b] = rec;
            }
        }
        __syncthreads(); // the bundle numbers of this chunk's first pushes
        if (p < ni && run_start) {
            const uint32_t b = __ldcg(dp.bord + i0 + bfirst);
            dp.run_item[i0 + r] = p;
            dp.run_bundle[i0 + r] = b;
            atomicAdd(dp.bcur + i0 + b, 1u);
        }
        carry = make_uint2(carry.x + total.x, carry.y + total.y);
        __syncthreads(); // this chunk's atomics before the counts are read
    }
    const uint32_t n_runs = carry.x, n_bundles = carry.y;
    // each run's last triangle: the run's items are consecutive pushes of one layout
    for (uint32_t p = t; p < ni; p += kBinThreads) {
        const uint32_t r = dp.run_of[i0 + p];
        if (p + 1u == ni || __ldcg(dp.run_of + i0 + p + 1u) != r) dp.run_tend[i0 + r] = dp.toff[i0 + p] + dp.items[dp.ord_item[i0 + p]].n_tris;
    }
    // 5. the bundles' instances: counts -> first instance (bcur becomes the cursor)
    __syncthreads();
    carry = make_uint2(0u, 0u);
    for (uint32_t b0 = 0; b0 < n_bundles; b0 += kBinThreads) {
        const uint32_t b = b0 + t;
        const uint32_t c = b < n_bundles ? __ldcg(dp.bcur + i0 + b) : 0u;
        const uint32_t first = carry.x + cta_exclusive_scan(make_uint2(c, 0u), total).x;
        if (b < n_bundles) {
            dp.bcur[i0 + b] = first;
            dp.o_bundles[i0 + b].first = first;
            dp.o_bundles[i0 + b].count = c;
        }
        carry.x += total.x;
    }
    __syncthreads(); // every bundle's first instance
    // each run's instance: its bundle's cursor before this chunk, plus the earlier runs of the same bundle in the chunk
    for (uint32_t r0 = 0; r0 < n_runs; r0 += kBinThreads) {
        const uint32_t r = r0 + t;
        const uint32_t b = r < n_runs ? __ldcg(dp.run_bundle + i0 + r) : FYX_NONE;
        s_b[t] = b;
        __syncthreads();
        if (r < n_runs) {
            uint32_t rank = 0u;
            for (uint32_t j = 0; j < t; ++j) rank += s_b[j] == b ? 1u : 0u;
            const uint32_t p = __ldcg(dp.run_item + i0 + r);
            const uint32_t tf = __ldcg(dp.toff + i0 + p);
            fyx_dynamic_instance inst;
            inst.node = dp.items[__ldcg(dp.ord_item + i0 + p)].node;
            inst.triangle_offset = tf;
            inst.triangle_count = __ldcg(dp.run_tend + i0 + r) - tf;
            inst.reserved = 0u;
            dp.o_inst[i0 + __ldcg(dp.bcur + i0 + b) + rank] = inst;
        }
        __syncthreads();
        if (r < n_runs) atomicAdd(dp.bcur + i0 + b, 1u);
        __syncthreads();
    }
    if (t == 0) {
        dp.o_seg[seg * 2] = n_bundles;
        dp.o_seg[seg * 2 + 1] = n_runs;
    }
}

// a float at any byte alignment
__device__ __forceinline__ float dyn_ld(const unsigned char *p)
{
    return __uint_as_float((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
}
__device__ __forceinline__ void dyn_st(unsigned char *p, const float f)
{
    const uint32_t u = __float_as_uint(f);
    p[0] = (unsigned char)u;
    p[1] = (unsigned char)(u >> 8);
    p[2] = (unsigned char)(u >> 16);
    p[3] = (unsigned char)(u >> 24);
}
// Matrix4::transform_point / transform_vector (nalgebra) of an affine world matrix, rows r0..r2, bottom row (0, 0, 0, 1):
// t = M3x3 * v (+ translation), n = row3 . v (+ 1); t / n unless n == 0 (scene/mesh/mod.rs:109-126)
__device__ __forceinline__ void dyn_transform(const float4 &r0, const float4 &r1, const float4 &r2, const float *v, const bool point, float *o)
{
    const float4 r[3] = {r0, r1, r2};
    float n = FYX_ADD(FYX_ADD(FYX_MUL(0.0f, v[0]), FYX_MUL(0.0f, v[1])), FYX_MUL(0.0f, v[2]));
    if (point) n = FYX_ADD(n, 1.0f);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float x = FYX_ADD(FYX_ADD(FYX_MUL(r[i].x, v[0]), FYX_MUL(r[i].y, v[1])), FYX_MUL(r[i].z, v[2]));
        if (point) x = FYX_ADD(x, r[i].w);
        o[i] = (n != 0.0f) ? __fdiv_rn(x, n) : x;
    }
}

// the segment of placed item q: the last whose first item is <= q
__device__ __forceinline__ uint32_t dyn_item_segment(const DynParams &dp, const uint32_t q)
{
    uint32_t lo = 0u, hi = dp.n_seg - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (dp.seg_item0[mid] <= q) lo = mid;
        else hi = mid - 1u;
    }
    return lo;
}

// geometry, one warp per registered surface: the vertex records copied (u32-wide when the stride allows), then the three
// attributes transformed by the node's world matrix; the triangles shifted by the item's first vertex in its stream.  Quad
// items are k_dyn_quads'.
__global__ void __launch_bounds__(kBlock) k_dyn_geometry(const NodeArrays a, const DynParams dp, const uint32_t n_items)
{
    const uint32_t q = (blockIdx.x * kBlock + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (q >= n_items) return;
    const DynItemDev it = dp.items[dp.ord_item[q]];
    if (it.kind != kDynMesh) return;
    const DynLayoutDev ly = dp.layouts[it.layout];
    const size_t sl = (size_t)dyn_item_segment(dp, q) * dp.n_layouts + it.layout;
    const uint32_t v0 = dp.voff[q];
    const unsigned char *src = dp.vtx + it.vtx_src;
    unsigned char *dst = dp.o_vtx + dp.stream_vtx[sl] + (size_t)v0 * ly.stride;
    const uint32_t bytes = it.n_verts * ly.stride;
    if ((ly.stride & 3u) == 0u) {
        for (uint32_t e = lane; e < bytes / 4u; e += 32u) reinterpret_cast<uint32_t *>(dst)[e] = reinterpret_cast<const uint32_t *>(src)[e];
    } else {
        for (uint32_t e = lane; e < bytes; e += 32u) dst[e] = src[e];
    }
    const uint32_t *ts = dp.tri + it.tri_src;
    uint32_t *td = dp.o_tri + ((size_t)dp.stream_tri[sl] + dp.toff[q]) * 3u;
    for (uint32_t e = lane; e < it.n_tris * 3u; e += 32u) td[e] = ts[e] + v0;
    __syncwarp();
    const float4 r0 = a.G[0][it.slot], r1 = a.G[1][it.slot], r2 = a.G[2][it.slot];
    for (uint32_t v = lane; v < it.n_verts; v += 32u) {
        const unsigned char *s = src + (size_t)v * ly.stride;
        unsigned char *d = dst + (size_t)v * ly.stride;
        float x[3], o[3];
        const uint32_t off[3] = {ly.pos, ly.nrm, ly.tan};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (off[k] == FYX_NONE) continue;
            x[0] = dyn_ld(s + off[k]);
            x[1] = dyn_ld(s + off[k] + 4);
            x[2] = dyn_ld(s + off[k] + 8);
            dyn_transform(r0, r1, r2, x, k == 0, o);
            dyn_st(d + off[k], o[0]);
            dyn_st(d + off[k] + 4, o[1]);
            dyn_st(d + off[k] + 8, o[2]);
        }
    }
}

// One vertex of a quad as words: SpriteVertex (10 words) or RectangleVertex (6 words), corner (sx, sy) = (+-0.5, +-0.5)
template <bool kSprite>
__device__ __forceinline__ void quad_vertex(const fyx_sprite &r, const float4 &r0, const float4 &r1, const float4 &r2, const float sx,
                                            const float sy, const float u, const float v, uint32_t *w)
{
    float p[3];
    if constexpr (kSprite) {
        p[0] = r0.w; // global_position(): the translation column, unchanged
        p[1] = r1.w;
        p[2] = r2.w;
    } else {
        const float c[3] = {sx, sy, 0.0f};
        dyn_transform(r0, r1, r2, c, true, p);
    }
    w[0] = __float_as_uint(p[0]);
    w[1] = __float_as_uint(p[1]);
    w[2] = __float_as_uint(p[2]);
    w[3] = __float_as_uint(u);
    w[4] = __float_as_uint(v);
    uint32_t k = 5;
    if constexpr (kSprite) {
        w[5] = __float_as_uint(r.size);
        w[6] = __float_as_uint(r.rotation);
        w[7] = __float_as_uint(sx);
        w[8] = __float_as_uint(sy);
        k = 9;
    }
    w[k] = (uint32_t)r.color[0] | ((uint32_t)r.color[1] << 8) | ((uint32_t)r.color[2] << 16) | ((uint32_t)r.color[3] << 24);
}

// The four vertices and two triangles of quad item q (scene/sprite.rs:331-379, scene/dim2/rectangle.rs:332-384).  The stream
// base is 16-byte aligned and both strides are multiples of 8: the vertices go out as 16-byte stores when the item's first
// vertex is even, else as 8-byte stores.
template <bool kSprite>
__device__ __forceinline__ void quad_write(const NodeArrays &a, const DynParams &dp, const DynItemDev &it, const uint32_t q)
{
    constexpr uint32_t kWords = kSprite ? 10u : 6u; // per vertex
    const fyx_sprite r = dp.quads[it.slot];
    const float4 r0 = a.G[0][it.slot], r1 = a.G[1][it.slot], r2 = a.G[2][it.slot];
    const float lx = r.uv_rect[0], rx = FYX_ADD(r.uv_rect[0], r.uv_rect[2]);
    const float ty = r.uv_rect[1], by = FYX_ADD(r.uv_rect[1], r.uv_rect[3]);
    const bool fx = r.flip & 1u, fy = r.flip & 2u;
    // corner k's tex_coord x is flip_x ? a : b with (a, b) = (lx, rx) for corners 0 and 3 of a sprite, 1 and 2 of a rectangle
    const float ua = fx ? lx : rx, ub = fx ? rx : lx;
    const float u[4] = {kSprite ? ua : ub, kSprite ? ub : ua, kSprite ? ub : ua, kSprite ? ua : ub};
    const float vt = fy ? by : ty, vb = fy ? ty : by;
    uint32_t w[4 * kWords];
    quad_vertex<kSprite>(r, r0, r1, r2, 0.5f, 0.5f, u[0], vt, w);
    quad_vertex<kSprite>(r, r0, r1, r2, -0.5f, 0.5f, u[1], vt, w + kWords);
    quad_vertex<kSprite>(r, r0, r1, r2, -0.5f, -0.5f, u[2], vb, w + 2 * kWords);
    quad_vertex<kSprite>(r, r0, r1, r2, 0.5f, -0.5f, u[3], vb, w + 3 * kWords);
    const size_t sl = (size_t)dyn_item_segment(dp, q) * dp.n_layouts + it.layout;
    const uint32_t v0 = dp.voff[q];
    unsigned char *dst = dp.o_vtx + dp.stream_vtx[sl] + (size_t)v0 * (kWords * 4u);
    if ((v0 & 1u) == 0u) {
#pragma unroll
        for (uint32_t k = 0; k < kWords; ++k) reinterpret_cast<uint4 *>(dst)[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
    } else {
#pragma unroll
        for (uint32_t k = 0; k < 2 * kWords; ++k) reinterpret_cast<uint2 *>(dst)[k] = make_uint2(w[2 * k], w[2 * k + 1]);
    }
    uint32_t *td = dp.o_tri + ((size_t)dp.stream_tri[sl] + dp.toff[q]) * 3u;
    td[0] = v0;
    td[1] = v0 + 1u;
    td[2] = v0 + 2u;
    td[3] = v0;
    td[4] = v0 + 2u;
    td[5] = v0 + 3u;
}

// quads, one thread per item; registered surfaces are k_dyn_geometry's
__global__ void __launch_bounds__(kBlock) k_dyn_quads(const NodeArrays a, const DynParams dp, const uint32_t n_items)
{
    const uint32_t q = blockIdx.x * kBlock + threadIdx.x;
    if (q >= n_items) return;
    const DynItemDev it = dp.items[dp.ord_item[q]];
    if (it.kind == FYX_SPRITE_3D) quad_write<true>(a, dp, it, q);
    else if (it.kind == FYX_SPRITE_RECTANGLE) quad_write<false>(a, dp, it, q);
}

} // namespace

// N3, bone matrices of the packed instances — RenderDataBundle::write_uniforms (renderer/bundle.rs:484-496): a skinned instance
// gets a block of MAX_BONE_MATRICES (255) mat4: its bone_matrices, then all-zero matrices; an unskinned one gets none.
// pass 1: which instance gets which block (order of the blocks is unspecified); inst_skin = the fyx surface id that skins the instance
__global__ void __launch_bounds__(kBlock) k_bone_block_index(const uint32_t n, const uint32_t *inst_skin, uint32_t *block_of_inst, uint32_t *counter)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i >= n) return;
    block_of_inst[i] = (inst_skin[i] != FYX_NONE) ? atomicAdd(counter, 1u) : FYX_NONE;
}
// pass 2: one CTA per instance (or, without inst_skin / block_of_inst, per surface: the shadow maps' blocks) copies the
// surface's palette and pads with zeros (1020 float4 per block)
__global__ void __launch_bounds__(kBlock) k_bone_blocks(const uint32_t *inst_skin, const uint2 *surf_bones /* (first palette entry, n_bones) */,
                                                        const float4 *palette, const uint32_t *block_of_inst, float4 *blocks)
{
    const uint32_t i = blockIdx.x;
    const uint32_t blk = block_of_inst ? block_of_inst[i] : i;
    if (blk == FYX_NONE) return;
    const uint2 sb = surf_bones[inst_skin ? inst_skin[i] : i];
    float4 *dst = blocks + (size_t)blk * (FYX_MAX_BONES * 4);
    const float4 *src = palette + (size_t)sb.x * 4;
    for (uint32_t e = threadIdx.x; e < FYX_MAX_BONES * 4; e += kBlock) dst[e] = (e < sb.y * 4u) ? src[e] : make_float4(0.f, 0.f, 0.f, 0.f);
}

void launch_bone_block_index(cudaStream_t s, uint32_t n, const uint32_t *inst_skin, uint32_t *block_of_inst, uint32_t *counter)
{
    if (n) k_bone_block_index<<<(n + kBlock - 1) / kBlock, kBlock, 0, s>>>(n, inst_skin, block_of_inst, counter);
}
void launch_bone_blocks(cudaStream_t s, uint32_t n, const uint32_t *inst_skin, const uint2 *surf_bones, const float *palette, const uint32_t *block_of_inst,
                        float *blocks)
{
    if (n) k_bone_blocks<<<n, kBlock, 0, s>>>(inst_skin, surf_bones, reinterpret_cast<const float4 *>(palette), block_of_inst, reinterpret_cast<float4 *>(blocks));
}

// the scratch is cleared by the caller: hist 0, first_key ~0 (segmented: seg_inst 0)
void launch_inst_count(cudaStream_t s, const NodeArrays &a, const InstParams &ip, bool segmented)
{
    const unsigned grid = (ip.n + kBlock - 1) / kBlock;
    if (!segmented) {
        if (ip.n) k_inst_keys<<<grid, kBlock, 0, s>>>(a, ip);
        k_inst_scan<<<1, kScanBlock, 0, s>>>(ip);
        return;
    }
    const uint32_t n_tiles = (ip.n_seg * ip.n_bundle_ids + kScanTile - 1) / kScanTile;
    if (ip.n) k_shadow_inst_keys<<<grid, kBlock, 0, s>>>(a, ip);
    launch_pdl(k_bin_reduce, n_tiles, kBinThreads, 0, s, ip);
    launch_pdl(k_bin_scan, 1, kBinThreads, 0, s, ip, n_tiles);
    launch_pdl(k_bin_downsweep, n_tiles, kBinThreads, 0, s, ip);
}

void launch_inst_scatter(cudaStream_t s, const NodeArrays &a, const InstParams &ip, bool segmented)
{
    if (!ip.n) return;
    const unsigned grid = (ip.n + kBlock - 1) / kBlock;
    if (segmented) k_shadow_inst_scatter<<<grid, kBlock, 0, s>>>(a, ip);
    else k_inst_scatter<<<grid, kBlock, 0, s>>>(a, ip);
}

void launch_dyn_mark(cudaStream_t s, const NodeArrays &a, const DynParams &dp)
{
    if (dp.n && dp.n_seg) k_dyn_mark<<<(dp.n + kBlock - 1) / kBlock, kBlock, 0, s>>>(a, dp);
}

int launch_dyn_batches(cudaStream_t s, const NodeArrays &a, const DynParams &dp, uint32_t n_items, bool meshes, bool quads)
{
    if (!n_items) return 0;
    k_dyn_order<<<dp.n_seg, kBinThreads, 0, s>>>(a, dp);
    if (meshes) k_dyn_geometry<<<(unsigned)(((uint64_t)n_items * 32u + kBlock - 1) / kBlock), kBlock, 0, s>>>(a, dp, n_items);
    if (quads) k_dyn_quads<<<(n_items + kBlock - 1) / kBlock, kBlock, 0, s>>>(a, dp, n_items);
    return 1 + (meshes ? 1 : 0) + (quads ? 1 : 0);
}

} // namespace fyx
