// fyx_kernels.cu — hand-written sm_90a kernels of the render-prep hot path.
//
// All kernels are HBM-bandwidth-bound streaming kernels over SoA planes (no tensor cores: 4x4 f32
// work at ~0.3-1 flop/B).  Arithmetic follows fyx_math.cuh (one rounding per op, reference order).
// Each kernel names the reference code it replaces (paths relative to the Fyrox tree).
#include <cuda_fp16.h>

#include "fyx_frustum.cuh"
#include "fyx_internal.h"
#include "fyx_trs.cuh"
#include "fyx_vcode.cuh"

namespace fyx {

// ------------------------------------------------------------------------------------------------
// streaming load/store helpers: node columns are touched once per frame ⇒ bypass L1 allocation for the
// big streams (read-only path, evict-first), keep default caching for the gathered parent rows.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_stream(const float4 *p)
{
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ float2 ld_stream(const float2 *p)
{
    float2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ld_stream(const uint4 *p)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream(float4 *p, const float4 v)
{
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void st_stream(float2 *p, const float2 v)
{
    asm volatile("st.global.L1::no_allocate.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
}

// ------------------------------------------------------------------------------------------------
// NodeTrait::should_be_rendered (scene/node/mod.rs:231-256) + the shadow-pass cast_shadows test of
// Mesh::collect_render_data (scene/mesh/mod.rs:696-698) + reachability from Graph::root
// (iterate_recursive, renderer/bundle.rs:988-1004), for every frustum of the call.  Bit f of the
// result = "node is in the visible set of frustum f".
// ------------------------------------------------------------------------------------------------
// NFT: number of frusta known at compile time (the loop is unrolled and cp.f[f] becomes constant-bank operands of the
// arithmetic instead of ~35 indexed parameter loads per frustum), 0 = run-time count.
// live: frusta whose geometric test this lane has to run.  Every caller passes all ones; the mask stays because without it
// ptxas allocates k_fold_bones differently (same results, different instructions).
constexpr uint32_t kNeedBits = FYX_NODE_ALIVE | FYX_NODE_RENDERABLE | FYX_NODE_REACHABLE | FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED;

template <int NFT>
__device__ __forceinline__ uint32_t cull_bits(const uint32_t nf, const uint32_t mask, const float2 wx, const float2 wy,
                                              const float2 wz, const CullParams &cp, const PackedConsts &kc, const bool tame, const uint32_t live)
{
    if ((nf & kNeedBits) != kNeedBits) return 0u;
    uint32_t bits = 0u;
    auto one = [&](const int f) {
        bool ok = (mask & cp.f[f].cam_mask) != 0u;
        ok &= !((cp.f[f].pass_flags & FYX_PASS_SHADOW) && !(nf & FYX_NODE_CAST_SHADOWS));
        if (ok && (nf & FYX_NODE_FRUSTUM_CULLING)) {
            if (((live >> f) & 1u) || !tame) ok = frustum_intersects_aabb(cp.f[f], wx, wy, wz, kc, tame);
            else ok = false;
        }
        bits |= ok ? (1u << f) : 0u;
    };
    if (NFT > 0) {
#pragma unroll
        for (int f = 0; f < NFT; ++f) one(f);
    } else {
        for (int f = 0; f < cp.nf; ++f) one(f);
    }
    return bits;
}

// Per-warp part of the cull, called by all 32 lanes: cand = this lane holds a node that may be emitted at all.
template <int NFT>
__device__ __forceinline__ uint32_t cull_warp(const bool cand, const uint32_t nf, const uint32_t mask, const float2 wx, const float2 wy,
                                              const float2 wz, const CullParams &cp)
{
    const PackedConsts kc = packed_consts(cp.one, cp.negzero);
    const bool ok = cand && (nf & kNeedBits) == kNeedBits;
    const bool tame = ok && aabb_is_tame(wx, wy, wz);
    return ok ? cull_bits<NFT>(nf, mask, wx, wy, wz, cp, kc, tame, 0xFFFFFFFFu) : 0u;
}

// ------------------------------------------------------------------------------------------------
// Compaction of the visible node indices.  Replaces the Vec pushes of RenderDataBundleStorage::push
// (renderer/bundle.rs:1248-1278).  Order inside a list is unspecified.  Two forms:
//  * CTA-wide (the level and cull kernels): warp ballot + popc rank, per-warp counts in shared memory, one atomicAdd per
//    (CTA, frustum);
//  * warp-wide (k_fold_bones, whose cull runs in warp 0 only): one atomicAdd per (warp, frustum that has a visible lane);
//    the counters sit on their own 128 B lines.
// Both must be called by every thread of the CTA / warp.
// ------------------------------------------------------------------------------------------------
template <int NFT>
__device__ __forceinline__ void compact_emit(const uint32_t vis_bits, const uint32_t node_index, const uint32_t slot,
                                             const CullParams &cp)
{
    constexpr int kWarps = kBlock / 32;
    __shared__ uint32_t s_wcount[FYX_MAX_FRUSTA][kWarps];
    __shared__ uint32_t s_base[FYX_MAX_FRUSTA];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nf = (NFT > 0) ? NFT : cp.nf;

    // any visible node in the CTA at all?  (most CTAs of a mostly-culled scene skip the atomics)
    const int any = __syncthreads_or(vis_bits != 0u);
    if (!any) return;

    for (int f = 0; f < nf; ++f) {
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, (vis_bits >> f) & 1u);
        if (lane == 0) s_wcount[f][warp] = __popc(b);
    }
    __syncthreads();
    if (threadIdx.x < nf) {
        const int f = threadIdx.x;
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
            const uint32_t c = s_wcount[f][w];
            s_wcount[f][w] = run; // exclusive prefix over warps
            run += c;
        }
        s_base[f] = run ? atomicAdd(cp.counts + f * kCountStride, run) : 0u;
    }
    __syncthreads();
    for (int f = 0; f < nf; ++f) {
        const uint32_t bit = (vis_bits >> f) & 1u;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, bit);
        if (bit) {
            const uint32_t pos = s_base[f] + s_wcount[f][warp] + __popc(b & ((1u << lane) - 1u));
            cp.out[f][pos] = node_index;
            if (cp.out_slot[f]) cp.out_slot[f][pos] = slot; // where the node lives in HBM (fyx_pack_instances)
        }
    }
}

__device__ __forceinline__ void compact_emit_warp(const uint32_t vis_bits, const uint32_t node_index, const uint32_t slot, const CullParams &cp)
{
    uint32_t m = __reduce_or_sync(0xFFFFFFFFu, vis_bits); // frusta with a visible lane in this warp (uniform)
    const uint32_t lane = threadIdx.x & 31u;
    while (m) {
        const int f = __ffs(m) - 1;
        m &= m - 1u;
        const uint32_t bit = (vis_bits >> f) & 1u;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, bit);
        uint32_t base = 0u;
        if (lane == 0) base = atomicAdd(cp.counts + f * kCountStride, (uint32_t)__popc(b));
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (bit) {
            const uint32_t pos = base + __popc(b & ((1u << lane) - 1u));
            cp.out[f][pos] = node_index;
            if (cp.out_slot[f]) cp.out_slot[f][pos] = slot;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// One hierarchy level.  Replaces, for the nodes of this level:
//   Graph::update_global_transform_recursively   scene/graph/mod.rs:1199-1241   (G = parent.G * local)
//   Graph::update_visibility_recursively          :1182-1197                      (gv = parent.gv && visibility)
//   Graph::update_enabled_flag_recursively        :1166-1180                      (ge = parent.ge && enabled)
//   Mesh::on_global_transform_changed / Base::world_bounding_box   scene/mesh/mod.rs:667-689, scene/base.rs:741-750
//   (+ (NFT >= 0): should_be_rendered + visible-list emission for non-skinned nodes)
// and the change tracking of process_node_messages (:1303-1399): a node is recomputed iff it or an
// ancestor changed (or FYX_UPDATE_ALL).  One thread per node; parents were finished by the previous
// launch on the same stream.
// Algorithmic bytes per node (SURVEY §8d): 132 (T) + 48 (A) [+ 8 (K)]; moved: 48+4+48 + 24+24 + 4+4(+4+4).
// ------------------------------------------------------------------------------------------------
// UA: FYX_UPDATE_ALL known at compile time — every load of the node's own columns is issued at once, next to the load of
// the parent index, instead of after the parent's flags have said whether the node is dirty (two dependent memory
// round trips per node instead of three).
template <bool WANT_BOX, bool UA>
__device__ __forceinline__ void update_node(const NodeArrays &a, const uint32_t slot, const uint32_t update_all, uint32_t &nf_out, float2 &wx,
                                            float2 &wy, float2 &wz)
{
    const uint32_t p = a.parent[slot]; // static column: may be read before the predecessor has finished
    pdl_wait(); // everything below reads what the previous level / a scatter kernel / the previous frame's tail wrote
    const uint32_t f = a.flags[slot]; // mutable (F_DIRTY_SELF is set by the scatter kernels): only after the wait
    Affine L;
    float2 lx, ly, lz;
    if (UA) {
        L.r0 = ld_stream(a.L[0] + slot);
        L.r1 = ld_stream(a.L[1] + slot);
        L.r2 = ld_stream(a.L[2] + slot);
        lx = ld_stream(a.la[0] + slot);
        ly = ld_stream(a.la[1] + slot);
        lz = ld_stream(a.la[2] + slot);
    }
    // no parent ⇒ parent values are identity / true (graph/mod.rs:1171-1175,1187-1192,1210-1214)
    const uint32_t pf = (p != FYX_NONE)
                            ? a.flags[p]
                            : (FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED | ((f & F_ROOT) ? FYX_NODE_REACHABLE : 0u));
    const bool dirty = UA || update_all || (f & F_DIRTY_SELF) || (pf & F_DIRTY);
    uint32_t nf = f & ~(FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED | FYX_NODE_REACHABLE | F_DIRTY | F_DIRTY_SELF);
    if ((pf & FYX_NODE_GLOBAL_VISIBILITY) && (f & FYX_NODE_VISIBILITY)) nf |= FYX_NODE_GLOBAL_VISIBILITY;
    if ((pf & FYX_NODE_GLOBAL_ENABLED) && (f & FYX_NODE_ENABLED)) nf |= FYX_NODE_GLOBAL_ENABLED;
    nf |= pf & FYX_NODE_REACHABLE;
    if (dirty) nf |= F_DIRTY;
    a.flags[slot] = nf;
    nf_out = nf;

    if (dirty) {
        if (!UA) {
            L.r0 = ld_stream(a.L[0] + slot);
            L.r1 = ld_stream(a.L[1] + slot);
            L.r2 = ld_stream(a.L[2] + slot);
            lx = ld_stream(a.la[0] + slot);
            ly = ld_stream(a.la[1] + slot);
            lz = ld_stream(a.la[2] + slot);
        }
        Affine P;
        if (p != FYX_NONE) {
            P.r0 = a.G[0][p]; // siblings are adjacent slots: one or two parents per warp (L1 hits)
            P.r1 = a.G[1][p];
            P.r2 = a.G[2][p];
        } else {
            P = affine_identity();
        }
        const Affine Gm = affine_mul(P, L);
        st_stream(a.G[0] + slot, Gm.r0);
        st_stream(a.G[1] + slot, Gm.r1);
        st_stream(a.G[2] + slot, Gm.r2);
        wx = aabb_transform_row(Gm.r0, lx, ly, lz);
        wy = aabb_transform_row(Gm.r1, lx, ly, lz);
        wz = aabb_transform_row(Gm.r2, lx, ly, lz);
        // skinned meshes: this is the box before the bone fold; fold_mesh finishes it
        st_stream(a.wa[0] + slot, wx);
        st_stream(a.wa[1] + slot, wy);
        st_stream(a.wa[2] + slot, wz);
    } else if (WANT_BOX) {
        wx = ld_stream(a.wa[0] + slot);
        wy = ld_stream(a.wa[1] + slot);
        wz = ld_stream(a.wa[2] + slot);
    }
}

// NFT < 0: no fused cull.  UA: FYX_UPDATE_ALL (update_node; the render mask and list index are loaded up front too).
template <int NFT, bool UA>
__global__ void __launch_bounds__(kBlock, 6) k_update_level(const NodeArrays a, const uint32_t lo, const uint32_t hi, const uint32_t update_all,
                                                            const CullParams cp)
{
    pdl_trigger();
    const uint32_t slot = lo + blockIdx.x * kBlock + threadIdx.x;
    uint32_t nf = 0u;
    float2 wx = make_float2(0.f, 0.f), wy = wx, wz = wx;
    const bool valid = slot < hi;
    uint32_t mask = 0u, gi_early = 0u;
    if (UA && (NFT >= 0) && valid) { // static columns: no reason to wait for anything
        mask = a.mask[slot];
        gi_early = a.gidx[slot];
    }
    if (valid) update_node<(NFT >= 0), UA>(a, slot, update_all, nf, wx, wy, wz);
    else pdl_wait();
    if (NFT >= 0) {
        const bool cand = valid && !(nf & F_SKINNED);
        if (!UA) mask = cand ? a.mask[slot] : 0u;
        const uint32_t vis_bits = cull_warp<(NFT > 0 ? NFT : 0)>(cand, nf, mask, wx, wy, wz, cp);
        const uint32_t gi = UA ? gi_early : (vis_bits ? a.gidx[slot] : 0u);
        compact_emit<(NFT > 0 ? NFT : 0)>(vis_bits, gi, slot, cp);
    }
}

// ------------------------------------------------------------------------------------------------
// The deep levels of the hierarchy in ONE launch (SubforestPlan, fyx_internal.h): a CTA owns a group of whole
// sub-trees — e.g. a dozen 64-bone skeletons — and walks their levels itself.  In every level the group's nodes are one
// contiguous slot range (coalesced like a level kernel); the matrices and flags of the previous level stay in shared
// memory for the children.  Same arithmetic, flags, change tracking and fused cull as k_update_level; what it removes
// is a kernel launch per level for levels of a few thousand nodes (C3: six skeleton levels of 10 k - 320 k nodes).
// ------------------------------------------------------------------------------------------------
template <int NFT, bool UA>
__global__ void __launch_bounds__(kBlock) k_update_subforest(const NodeArrays a, const uint2 *__restrict__ rng, const int n_levels,
                                                             const uint32_t update_all, const CullParams cp)
{
    pdl_trigger();
    __shared__ float4 s_g[2][3][kSfCap];
    __shared__ uint32_t s_f[2][kSfCap];
    const uint2 *my = rng + (size_t)blockIdx.x * n_levels;
    pdl_wait();
    uint32_t prevA = 0u, prevB = 0u;
    for (int li = 0; li < n_levels; ++li) {
        const uint2 r = my[li];
        const int cur = li & 1, prv = cur ^ 1;
        for (uint32_t base = r.x; base < r.y; base += kBlock) { // the same trip count for every thread of the CTA
            const uint32_t slot = base + threadIdx.x;
            const bool valid = slot < r.y;
            uint32_t nf = 0u;
            float2 wx = make_float2(0.f, 0.f), wy = wx, wz = wx;
            if (valid) {
                const uint32_t p = a.parent[slot];
                const uint32_t f = a.flags[slot];
                Affine L;
                float2 lx, ly, lz;
                if (UA) {
                    L.r0 = ld_stream(a.L[0] + slot);
                    L.r1 = ld_stream(a.L[1] + slot);
                    L.r2 = ld_stream(a.L[2] + slot);
                    lx = ld_stream(a.la[0] + slot);
                    ly = ld_stream(a.la[1] + slot);
                    lz = ld_stream(a.la[2] + slot);
                }
                const bool in_prev = (li > 0) && (p >= prevA) && (p < prevB); // the parent was handled by this CTA one level up
                const uint32_t pf = in_prev ? s_f[prv][p - prevA]
                                            : ((p != FYX_NONE) ? a.flags[p]
                                                               : (FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED | ((f & F_ROOT) ? FYX_NODE_REACHABLE : 0u)));
                const bool dirty = UA || update_all || (f & F_DIRTY_SELF) || (pf & F_DIRTY);
                nf = f & ~(FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED | FYX_NODE_REACHABLE | F_DIRTY | F_DIRTY_SELF);
                if ((pf & FYX_NODE_GLOBAL_VISIBILITY) && (f & FYX_NODE_VISIBILITY)) nf |= FYX_NODE_GLOBAL_VISIBILITY;
                if ((pf & FYX_NODE_GLOBAL_ENABLED) && (f & FYX_NODE_ENABLED)) nf |= FYX_NODE_GLOBAL_ENABLED;
                nf |= pf & FYX_NODE_REACHABLE;
                if (dirty) nf |= F_DIRTY;
                a.flags[slot] = nf;
                const uint32_t me = slot - r.x;
                s_f[cur][me] = nf;
                Affine Gm;
                if (dirty) {
                    if (!UA) {
                        L.r0 = ld_stream(a.L[0] + slot);
                        L.r1 = ld_stream(a.L[1] + slot);
                        L.r2 = ld_stream(a.L[2] + slot);
                        lx = ld_stream(a.la[0] + slot);
                        ly = ld_stream(a.la[1] + slot);
                        lz = ld_stream(a.la[2] + slot);
                    }
                    Affine P;
                    if (in_prev) {
                        P.r0 = s_g[prv][0][p - prevA];
                        P.r1 = s_g[prv][1][p - prevA];
                        P.r2 = s_g[prv][2][p - prevA];
                    } else if (p != FYX_NONE) {
                        P.r0 = a.G[0][p];
                        P.r1 = a.G[1][p];
                        P.r2 = a.G[2][p];
                    } else {
                        P = affine_identity();
                    }
                    Gm = affine_mul(P, L);
                    st_stream(a.G[0] + slot, Gm.r0);
                    st_stream(a.G[1] + slot, Gm.r1);
                    st_stream(a.G[2] + slot, Gm.r2);
                    wx = aabb_transform_row(Gm.r0, lx, ly, lz);
                    wy = aabb_transform_row(Gm.r1, lx, ly, lz);
                    wz = aabb_transform_row(Gm.r2, lx, ly, lz);
                    st_stream(a.wa[0] + slot, wx);
                    st_stream(a.wa[1] + slot, wy);
                    st_stream(a.wa[2] + slot, wz);
                } else {
                    // clean node: its children may be dirty and need its (unchanged) matrix
                    Gm.r0 = a.G[0][slot];
                    Gm.r1 = a.G[1][slot];
                    Gm.r2 = a.G[2][slot];
                    if (NFT >= 0) {
                        wx = ld_stream(a.wa[0] + slot);
                        wy = ld_stream(a.wa[1] + slot);
                        wz = ld_stream(a.wa[2] + slot);
                    }
                }
                s_g[cur][0][me] = Gm.r0;
                s_g[cur][1][me] = Gm.r1;
                s_g[cur][2][me] = Gm.r2;
            }
            if (NFT >= 0) {
                const bool cand = valid && !(nf & F_SKINNED);
                const uint32_t mask = cand ? a.mask[slot] : 0u;
                const uint32_t vis_bits = cull_warp<(NFT > 0 ? NFT : 0)>(cand, nf, mask, wx, wy, wz, cp);
                const uint32_t gi = vis_bits ? a.gidx[slot] : 0u;
                compact_emit<(NFT > 0 ? NFT : 0)>(vis_bits, gi, slot, cp);
            }
        }
        __syncthreads(); // this level's rows are complete (and the previous level's are no longer read)
        prevA = r.x;
        prevB = r.y;
    }
}

// ------------------------------------------------------------------------------------------------
// Stand-alone cull over all slots (static scene / extra passes: every shadow pass re-runs the cull
// with its own frustum, renderer/shadow/*.rs).  32 B read per node + 4 B per visible entry.
// ------------------------------------------------------------------------------------------------
// the node's row of a pruner table: its own (it is a pruner) or its nearest pruner ancestor's children row
__device__ __forceinline__ const uint32_t *pruner_row(const uint32_t *rows, const uint32_t words, const uint32_t pc)
{
    if (pc == FYX_NONE) return nullptr;
    return rows + ((size_t)(pc & ~kPrSelf) * 2u + ((pc & kPrSelf) ? 0u : 1u)) * words;
}

// One step of a pruner table, for pruner p at `slot` and the maps [32 w, 32 w + 32) of n_maps — the pruned DFS of
// renderer/bundle.rs:898-916, 988-1004 with each map's observer, and Mesh::collect_render_data's Break
// (scene/mesh/mod.rs:691-725):
//   self_hidden[p]     = children_hidden[anc(p)] | (LOD object outside its range for the map's observer)
//   children_hidden[p] = self_hidden[p] | (static batch drawn in the map)
// Every pruner table computes its rows here; the caller gives map m's LOD observer, observer(m) (a fyx_observer: the
// translation, z_near and z_far of ObserverPosition), and drawn(m): the node is in map m's list.
template <class Observer, class Drawn>
__device__ __forceinline__ void pruner_step(const NodeArrays &a, const MapParams::Prune &pr, const uint32_t p, const uint32_t slot,
                                            const uint32_t w, const uint32_t n_maps, Observer observer, Drawn drawn)
{
    const uint32_t W = pr.words, anc = pr.anc[p];
    uint32_t self = anc != FYX_NONE ? pr.rows[((size_t)anc * 2u + 1u) * W + w] : 0u, rendered = 0u;
    const float2 r = pr.range ? pr.range[slot] : make_float2(NAN, NAN);
    const bool lod = r.x == r.x, batch = (a.flags[slot] & FYX_NODE_STATIC_BATCH) != 0u;
    const float gx = a.G[0][slot].w, gy = a.G[1][slot].w, gz = a.G[2][slot].w; // global_position()
    for (uint32_t b = 0; b < 32u; ++b) {
        const uint32_t m = w * 32u + b;
        if (m >= n_maps) break;
        if (lod) { // metric_distance: |observer - position|, nalgebra's left-to-right dot, then sqrt
            const fyx_observer o = observer(m);
            const float dx = FYX_ADD(o.translation[0], -gx), dy = FYX_ADD(o.translation[1], -gy), dz = FYX_ADD(o.translation[2], -gz);
            const float dist = __fsqrt_rn(FYX_ADD(FYX_ADD(FYX_MUL(dx, dx), FYX_MUL(dy, dy)), FYX_MUL(dz, dz)));
            const float normalized = __fdiv_rn(FYX_ADD(dist, -o.z_near), FYX_ADD(o.z_far, -o.z_near));
            if (!((normalized >= r.x) && (normalized <= r.y))) self |= 1u << b;
        }
        if (batch && drawn(m)) rendered |= 1u << b;
    }
    pr.rows[((size_t)p * 2u) * W + w] = self;
    pr.rows[((size_t)p * 2u + 1u) * W + w] = self | rendered;
}

// The pruner table of a camera cull, one launch per hierarchy level's pruners [p_lo, p_hi) (parents first), one thread per
// pruner and one word per row (at most FYX_MAX_FRUSTA frusta); drawn in frustum f = bit f of cull_bits, k_cull's predicate.
// The LOD observers travel by value (pr.range nullptr: no LOD filter, obs unused).
__global__ void __launch_bounds__(kBlock) k_cull_pruners(const NodeArrays a, const CullParams cp, const MapParams::Prune pr, const Observers obs,
                                                         const uint32_t p_lo, const uint32_t p_hi)
{
    const uint32_t p = p_lo + blockIdx.x * kBlock + threadIdx.x;
    if (p >= p_hi) return;
    const uint32_t slot = pr.slot[p];
    const uint32_t drawn = cull_warp<0>(true, a.flags[slot], a.mask[slot], a.wa[0][slot], a.wa[1][slot], a.wa[2][slot], cp);
    pruner_step(a, pr, p, slot, 0u, (uint32_t)cp.nf, [&](const uint32_t m) { return obs.o[m]; },
                [&](const uint32_t m) { return ((drawn >> m) & 1u) != 0u; });
}

// pr.col != nullptr: a node is hidden for the frusta in which its row of the camera's pruner table (k_cull_pruners, one word
// per row) says the DFS stopped above it or at it: a LOD object out of range, or a statically batched mesh that is rendered
// (RdcControlFlow::Break, scene/mesh/mod.rs:725; renderer/bundle.rs:996-1001).
template <int NFT>
__global__ void __launch_bounds__(kBlock) k_cull(const NodeArrays a, const CullParams cp, const MapParams::Prune pr)
{
    const uint32_t slot = blockIdx.x * kBlock + threadIdx.x;
    const bool valid = slot < a.cap;
    uint32_t nf = 0u, mask = 0u;
    float2 wx = make_float2(0.f, 0.f), wy = wx, wz = wx;
    if (valid) {
        nf = a.flags[slot];
        mask = a.mask[slot];
        wx = ld_stream(a.wa[0] + slot);
        wy = ld_stream(a.wa[1] + slot);
        wz = ld_stream(a.wa[2] + slot);
    }
    uint32_t vis_bits = cull_warp<NFT>(valid, nf, mask, wx, wy, wz, cp);
    if (pr.col && vis_bits) {
        const uint32_t *row = pruner_row(pr.rows, 1u, pr.col[slot]);
        if (row) vis_bits &= ~*row;
    }
    const uint32_t gi = vis_bits ? a.gidx[slot] : 0u;
    compact_emit<NFT>(vis_bits, gi, slot, cp);
}

// ------------------------------------------------------------------------------------------------
// Light list (N4): the collect_lights loop of RenderDataBundleStorage::from_graph (renderer/bundle.rs:926-974) — for every
// frustum the light nodes whose world box it intersects and that are globally visible and enabled.  Lights are few:
// one pass over the flag column (4 B/node), one atomic per visible (light, frustum).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_cull_lights(const NodeArrays a, const CullParams cp, uint32_t *const *out, uint32_t *counts)
{
    const uint32_t slot = blockIdx.x * kBlock + threadIdx.x;
    if (slot >= a.cap) return;
    const uint32_t nf = a.flags[slot];
    constexpr uint32_t need = FYX_NODE_ALIVE | FYX_NODE_LIGHT | FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED;
    if ((nf & need) != need) return;
    const float2 wx = a.wa[0][slot], wy = a.wa[1][slot], wz = a.wa[2][slot];
    const PackedConsts kc = packed_consts(cp.one, cp.negzero);
    const bool tame = aabb_is_tame(wx, wy, wz);
    const uint32_t gi = a.gidx[slot];
    for (int f = 0; f < cp.nf; ++f)
        if (frustum_intersects_aabb(cp.f[f], wx, wy, wz, kc, tame)) out[f][atomicAdd(counts + f * kCountStride, 1u)] = gi;
}

// ------------------------------------------------------------------------------------------------
// Skinned-mesh world AABB: the "special case for skinned meshes" of Mesh::on_global_transform_changed
// (scene/mesh/mod.rs:673-684): world_aabb.add_point(bone.global_position()) for every bone of every
// surface, strict </> updates in bone order (aabb.rs:86-106).  Runs after all levels (bones may be deeper than the mesh node);
// only meshes in a changed sub-tree are refreshed, as in the reference.  With (NFT >= 0) the skinned
// nodes are also culled here (they were skipped by the level kernels).
// ------------------------------------------------------------------------------------------------
// One WARP per skinned mesh: lanes take the bones round-robin, then the per-lane candidates are merged with
// a shuffle reduction keyed (value, position in the bone list) so that among numerically equal bounds
// (only -0 / +0 can differ in bits) the first one in the reference's order wins — the result is the
// reference's sequential add_point loop, bit for bit.
__device__ __forceinline__ void fold_min(float &v, uint32_t &k, const float ov, const uint32_t ok)
{
    if (ov < v || (ov == v && ok < k)) { v = ov; k = ok; }
}
__device__ __forceinline__ void fold_max(float &v, uint32_t &k, const float ov, const uint32_t ok)
{
    if (ov > v || (ov == v && ok < k)) { v = ov; k = ok; }
}

// one warp = one skinned mesh (i): refreshes the world box (all lanes return it) and reads what the cull needs
// Every table load that does not depend on another one is issued up front (mesh slot, bone range, the first two rounds of
// bone slots): three dependent memory round trips per mesh (index -> bone slot -> bone matrix) instead of five.
__device__ __forceinline__ void fold_mesh(const NodeArrays &a, const FoldArrays &fa, const uint32_t i, const uint32_t lane, uint32_t &nf_out,
                                          float2 &wx, float2 &wy, float2 &wz)
{
    const uint32_t slot = fa.node_slot[i];
    const uint32_t b0 = fa.bone_begin[i], b1 = fa.bone_begin[i + 1];
    uint32_t bs_pre[2], si_pre[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const uint32_t b = b0 + lane + 32u * r;
        bs_pre[r] = (b < b1) ? fa.bone_slot[b] : FYX_NONE;
        si_pre[r] = (b < b1 && fa.stale_idx) ? fa.stale_idx[b] : FYX_NONE;
    }
    const uint32_t nf = a.flags[slot];
    nf_out = nf;
    wx = a.wa[0][slot];
    wy = a.wa[1][slot];
    wz = a.wa[2][slot];
    if (!(nf & F_DIRTY)) return;
    // candidates start as the transformed box (order key 0 = "already there"); bones get keys 1..
    float mnx = wx.x, mny = wy.x, mnz = wz.x, mxx = wx.y, mxy = wy.y, mxz = wz.y;
    uint32_t kmnx = 0, kmny = 0, kmnz = 0, kmxx = 0, kmxy = 0, kmxz = 0;
    auto add_bone = [&](const uint32_t b, const uint32_t bs, const uint32_t si) {
        if (bs == FYX_NONE) return; // try_borrow failed ⇒ skipped
        float px, py, pz; // global_position()
        if (si != FYX_NONE) { // visited after the mesh by the reference's DFS: its value from before this update
            const float4 o = fa.stale_pos[si];
            px = o.x; py = o.y; pz = o.z;
        } else {
            px = a.G[0][bs].w;
            py = a.G[1][bs].w;
            pz = a.G[2][bs].w;
        }
        const uint32_t key = b - b0 + 1u;
        // within a lane keys increase, so the strict compares keep the earliest of equal values
        if (px < mnx) { mnx = px; kmnx = key; }
        if (py < mny) { mny = py; kmny = key; }
        if (pz < mnz) { mnz = pz; kmnz = key; }
        if (px > mxx) { mxx = px; kmxx = key; }
        if (py > mxy) { mxy = py; kmxy = key; }
        if (pz > mxz) { mxz = pz; kmxz = key; }
    };
#pragma unroll
    for (int r = 0; r < 2; ++r) add_bone(b0 + lane + 32u * r, bs_pre[r], si_pre[r]);
    for (uint32_t b = b0 + lane + 64u; b < b1; b += 32)
        add_bone(b, fa.bone_slot[b], fa.stale_idx ? fa.stale_idx[b] : FYX_NONE);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        fold_min(mnx, kmnx, __shfl_xor_sync(0xFFFFFFFFu, mnx, o), __shfl_xor_sync(0xFFFFFFFFu, kmnx, o));
        fold_min(mny, kmny, __shfl_xor_sync(0xFFFFFFFFu, mny, o), __shfl_xor_sync(0xFFFFFFFFu, kmny, o));
        fold_min(mnz, kmnz, __shfl_xor_sync(0xFFFFFFFFu, mnz, o), __shfl_xor_sync(0xFFFFFFFFu, kmnz, o));
        fold_max(mxx, kmxx, __shfl_xor_sync(0xFFFFFFFFu, mxx, o), __shfl_xor_sync(0xFFFFFFFFu, kmxx, o));
        fold_max(mxy, kmxy, __shfl_xor_sync(0xFFFFFFFFu, mxy, o), __shfl_xor_sync(0xFFFFFFFFu, kmxy, o));
        fold_max(mxz, kmxz, __shfl_xor_sync(0xFFFFFFFFu, mxz, o), __shfl_xor_sync(0xFFFFFFFFu, kmxz, o));
    }
    wx = make_float2(mnx, mxx);
    wy = make_float2(mny, mxy);
    wz = make_float2(mnz, mxz);
    if (lane == 0) {
        a.wa[0][slot] = wx;
        a.wa[1][slot] = wy;
        a.wa[2][slot] = wz;
    }
}

// One warp per skinned mesh folds the bones; the cull of the CTA's kBlock/32 meshes is then run by the first lanes of warp 0,
// one mesh per LANE (the multi-frustum predicate is a long dependent chain: run by lane 0 of every warp it cost eight times the
// issue slots), and warp 0 emits the entries.
template <int NFT>
__global__ void __launch_bounds__(kBlock) k_fold_bones(const NodeArrays a, const FoldArrays fa, const CullParams cp)
{
    pdl_trigger();
    pdl_wait();
    constexpr int kWarps = kBlock / 32;
    __shared__ float2 s_box[3][kWarps];
    __shared__ uint32_t s_nf[kWarps];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t i = blockIdx.x * kWarps + warp; // mesh = warp
    uint32_t nf = 0u;
    float2 wx = make_float2(0.f, 0.f), wy = wx, wz = wx;
    if (i < fa.n) fold_mesh(a, fa, i, lane, nf, wx, wy, wz);
    if (NFT < 0) return;
    if (lane == 0) {
        s_box[0][warp] = wx;
        s_box[1][warp] = wy;
        s_box[2][warp] = wz;
        s_nf[warp] = (i < fa.n) ? nf : 0u;
    }
    __syncthreads();
    if (warp != 0) return;
    uint32_t vis_bits = 0u, gi = 0u, slot = 0u;
    const uint32_t m = blockIdx.x * kWarps + lane; // lane l of warp 0 culls the mesh of warp l
    if (lane < kWarps && m < fa.n) {
        const PackedConsts kc = packed_consts(cp.one, cp.negzero);
        slot = fa.node_slot[m];
        const float2 bx = s_box[0][lane], by = s_box[1][lane], bz = s_box[2][lane];
        vis_bits = cull_bits<(NFT > 0 ? NFT : 0)>(s_nf[lane], a.mask[slot], bx, by, bz, cp, kc, aabb_is_tame(bx, by, bz), 0xFFFFFFFFu);
        if (vis_bits) gi = a.gidx[slot];
    }
    compact_emit_warp(vis_bits, gi, slot, cp);
}

// positions of the "late" bones (see FoldArrays) as stored before the update starts
__global__ void __launch_bounds__(kBlock) k_snapshot_bones(const NodeArrays a, const uint32_t n_late, const uint32_t *late_slot,
                                                           float4 *stale_pos)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= n_late) return;
    const uint32_t s = late_slot[e];
    stale_pos[e] = make_float4(a.G[0][s].w, a.G[1][s].w, a.G[2][s].w, 0.0f);
}

// ------------------------------------------------------------------------------------------------
// Bone palette: SurfaceInstanceData::bone_matrices (scene/mesh/mod.rs:781-793):
// P[k] = bone_k.global_transform() * bone_k.inv_bind_pose_transform(), identity for an invalid
// handle.  One thread per (surface, bone) entry; G is gathered by bone slot, inv_bind streams.
// Output: column-major mat4 (the layout write_uniforms copies into the UBO, renderer/bundle.rs:484-496).
// Algorithmic bytes per bone: 196 (G 64 + inv_bind 64 + idx 4 + P 64); moved: 48 + 48 + 4 + 64.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void palette_entry(const NodeArrays &a, const SkinArrays &sk, const uint32_t e)
{
    const uint32_t bs = sk.bone_slot[e];
    Affine P;
    if (bs != FYX_NONE) {
        Affine Gm, IB;
        Gm.r0 = a.G[0][bs];
        Gm.r1 = a.G[1][bs];
        Gm.r2 = a.G[2][bs];
        IB.r0 = ld_stream(sk.ib[0] + e);
        IB.r1 = ld_stream(sk.ib[1] + e);
        IB.r2 = ld_stream(sk.ib[2] + e);
        P = affine_mul(Gm, IB);
    } else {
        P = affine_identity();
    }
    float4 *o = reinterpret_cast<float4 *>(sk.palette + 16 * (size_t)e);
    o[0] = make_float4(P.r0.x, P.r1.x, P.r2.x, 0.0f);
    o[1] = make_float4(P.r0.y, P.r1.y, P.r2.y, 0.0f);
    o[2] = make_float4(P.r0.z, P.r1.z, P.r2.z, 0.0f);
    o[3] = make_float4(P.r0.w, P.r1.w, P.r2.w, 1.0f);
}

__global__ void __launch_bounds__(kBlock) k_palette(const NodeArrays a, const SkinArrays sk)
{
    pdl_trigger();
    pdl_wait();
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e < sk.n_entries) palette_entry(a, sk, e);
}

// ------------------------------------------------------------------------------------------------
// Linear-blend skinning.  Positions: the skinned branch of Mesh::accurate_world_bounding_box
// (scene/mesh/mod.rs:501-522): acc = 0; for k in 0..4: acc += P[idx_k].transform_point(p) * w_k, where
// transform_point = ((m_i0*x + m_i1*y) + m_i2*z) + m_i3, then / n with n = row3·p + m33 — exactly 1
// for the affine palette and finite p, so the division is the identity and is skipped.  Normals:
// standard.shader:192-195, acc += (mat3(P[idx_k]) * n) * w_k in the same order.
//
// * Each thread owns 4 consecutive vertices.  Inputs live in blocks of 128 vertices x 11 rows of 512 B
//   (x, y, z, nx, ny, nz, w0..w3, indices; fyx_internal.h): a warp reads a row with ONE coalesced 512 B
//   access and each 32 B sector exactly once (the packed-xyz layout made every sector travel L2->SM
//   twice).  Outputs are packed xyz streams, 3 + 3 128-bit stores per thread.
// * Arithmetic is written on pairs (mul2 / add2, fyx_math.cuh: one rounding per element; sm_90 issues
//   each element as its own FMUL / FADD).  Pairs: (x,y) of the position, (x,y) of the normal, and
//   (position.z, normal.z) — same op order per element as the scalar reference.
// * The surface's palette sits in shared memory as three float4 planes laid out for those pairs:
//     A = (m00,m10,m01,m11)  B = (m02,m12,m03,m13)  Z = (m20,m21,m22,m23)
//   (the z pair multiplies the register pair (p,n) by a broadcast coefficient, so the third
//   row needs no duplication), each plane REPLICATED C times: bone b of copy c at float4 index plane*PL + c*S + b with S = 1 mod 8,
//   PL = C*S.  A 128-bit shared load is served per quarter-warp; lane l reads copy (l - b) mod C,
//   which puts it in bank group (plane*PL + l) mod 8: conflict-free for C = 8 whatever the bone
//   indices are (with one copy, lanes that read the same bank group collide).
// Algorithmic bytes per vertex: 44 read + 24 written = 68.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 lo2(const float4 v) { return make_float2(v.x, v.y); }
__device__ __forceinline__ float2 hi2(const float4 v) { return make_float2(v.z, v.w); }

// palette (column-major mat4 in global memory) → the four replicated planes
template <int S, int LOG2C>
__device__ __forceinline__ void skin_fill_palette(float4 *s_pal, const float *palette, const uint32_t bone_off, const uint32_t n_bones)
{
    constexpr int C = 1 << LOG2C;
    constexpr int PL = S * C;
    for (uint32_t b = threadIdx.x; b < n_bones; b += kBlock) {
        const float4 *m = reinterpret_cast<const float4 *>(palette + 16 * (size_t)(bone_off + b));
        const float4 c0 = m[0], c1 = m[1], c2 = m[2], c3 = m[3];
        const float4 A = make_float4(c0.x, c0.y, c1.x, c1.y);
        const float4 B = make_float4(c2.x, c2.y, c3.x, c3.y);
        const float4 Z = make_float4(c0.z, c1.z, c2.z, c3.z);
#pragma unroll
        for (int c = 0; c < C; ++c) {
            s_pal[0 * PL + c * S + b] = A;
            s_pal[1 * PL + c * S + b] = B;
            s_pal[2 * PL + c * S + b] = Z;
        }
    }
}

// four vertices (one thread's group) from registers to their packed xyz outputs, 3 float4 per stream
template <int S, int LOG2C>
__device__ __forceinline__ void skin_quad_regs(const float4 *s_pal, const uint32_t lane, const float4 x4, const float4 y4, const float4 z4,
                                               const float4 nx4, const float4 ny4, const float4 nz4, const float4 w0, const float4 w1,
                                               const float4 w2, const float4 w3, const uint4 iq, float4 (&po)[3], float4 (&no)[3],
                                               const PackedConsts kc)
{
    constexpr int C = 1 << LOG2C;
    constexpr int PL = S * C;
    const float px[4] = {x4.x, x4.y, x4.z, x4.w}, py[4] = {y4.x, y4.y, y4.z, y4.w}, pz[4] = {z4.x, z4.y, z4.z, z4.w};
    const float nx[4] = {nx4.x, nx4.y, nx4.z, nx4.w}, ny[4] = {ny4.x, ny4.y, ny4.z, ny4.w}, nz[4] = {nz4.x, nz4.y, nz4.z, nz4.w};
    // w_k holds weight k of the four vertices
    const float wk4[4][4] = {{w0.x, w1.x, w2.x, w3.x}, {w0.y, w1.y, w2.y, w3.y}, {w0.z, w1.z, w2.z, w3.z}, {w0.w, w1.w, w2.w, w3.w}};
    const uint32_t iv[4] = {iq.x, iq.y, iq.z, iq.w};
    float ox[4], oy[4], oz[4], mx[4], my[4], mz[4];
#pragma unroll
    for (int v = 0; v < 4; ++v) {
        const float2 pxx = make_float2(px[v], px[v]), pyy = make_float2(py[v], py[v]), pzz = make_float2(pz[v], pz[v]);
        const float2 nxx = make_float2(nx[v], nx[v]), nyy = make_float2(ny[v], ny[v]), nzz = make_float2(nz[v], nz[v]);
        const float2 pnx = make_float2(px[v], nx[v]), pny = make_float2(py[v], ny[v]), pnz = make_float2(pz[v], nz[v]);
        float2 acc_p = make_float2(0.0f, 0.0f), acc_n = make_float2(0.0f, 0.0f), acc_z = make_float2(0.0f, 0.0f);
        const float *wk = wk4[v];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t bone = (iv[v] >> (8 * k)) & 0xFFu;
            const float4 *row = s_pal + (((lane - bone) & (uint32_t)(C - 1)) * S + bone);
            const float4 A = row[0], B = row[PL], Z = row[2 * PL];
            const float2 ww = make_float2(wk[k], wk[k]);
            // (tx, ty) = ((m_i0*x + m_i1*y) + m_i2*z) + m_i3, i = 0,1
            const float2 t = add2(add2(add2(mul2(lo2(A), pxx, kc), mul2(hi2(A), pyy, kc), kc), mul2(lo2(B), pzz, kc), kc), hi2(B), kc);
            acc_p = add2(acc_p, mul2(t, ww, kc), kc);
            // (rx, ry) = (m_i0*nx + m_i1*ny) + m_i2*nz
            const float2 r = add2(add2(mul2(lo2(A), nxx, kc), mul2(hi2(A), nyy, kc), kc), mul2(lo2(B), nzz, kc), kc);
            acc_n = add2(acc_n, mul2(r, ww, kc), kc);
            // (tz', rz) = (m_20*{x,nx} + m_21*{y,ny}) + m_22*{z,nz};  tz = tz' + m_23
            float2 z = add2(add2(mul2(pnx, make_float2(Z.x, Z.x), kc), mul2(pny, make_float2(Z.y, Z.y), kc), kc), mul2(pnz, make_float2(Z.z, Z.z), kc), kc);
            z.x = FYX_ADD(z.x, Z.w);
            acc_z = add2(acc_z, mul2(z, ww, kc), kc);
        }
        ox[v] = acc_p.x; oy[v] = acc_p.y; oz[v] = acc_z.x;
        mx[v] = acc_n.x; my[v] = acc_n.y; mz[v] = acc_z.y;
    }
    po[0] = make_float4(ox[0], oy[0], oz[0], ox[1]);
    po[1] = make_float4(oy[1], oz[1], ox[2], oy[2]);
    po[2] = make_float4(oz[2], ox[3], oy[3], oz[3]);
    no[0] = make_float4(mx[0], my[0], mz[0], mx[1]);
    no[1] = make_float4(my[1], mz[1], mx[2], my[2]);
    no[2] = make_float4(mz[2], mx[3], my[3], mz[3]);
}

// N4: blend shapes ahead of the skinning (standard.shader:167-173): for i in 0..blendShapesCount:
//   inputPosition.xyz += offsets.position * weight;  inputNormal += offsets.normal * weight
// in shape order, offsets = the f16 texels of BlendShapesContainer::from_lists (scene/mesh/surface.rs:92-218, exact in
// f32), weight = BlendShape::weight / 100 (scene/mesh/mod.rs:794-798); one rounding per product and per sum.
// 12 more bytes read per vertex and shape.  The four vertices of a thread come as 4 halfs per row.
__device__ __forceinline__ void bs_axpy(float4 &v, const uint2 h, const float w)
{
    const __half2 a = *reinterpret_cast<const __half2 *>(&h.x), b = *reinterpret_cast<const __half2 *>(&h.y);
    const float2 fa = __half22float2(a), fb = __half22float2(b);
    v.x = FYX_ADD(v.x, FYX_MUL(fa.x, w));
    v.y = FYX_ADD(v.y, FYX_MUL(fa.y, w));
    v.z = FYX_ADD(v.z, FYX_MUL(fb.x, w));
    v.w = FYX_ADD(v.w, FYX_MUL(fb.y, w));
}

__device__ __forceinline__ void apply_blend_shapes(const SkinArrays &sk, const SkinTile &T, const uint32_t q, float4 &x4, float4 &y4, float4 &z4,
                                                   float4 &nx4, float4 &ny4, float4 &nz4)
{
    const uint32_t e = T.local_quad0 + q;
    const uint2 *r0 = sk.bs + ((size_t)T.bs_off + (e >> 5)) * kBsBlockU2 + (e & 31u);
    const size_t shape_stride = (size_t)T.bs_blocks * kBsBlockU2;
    for (uint32_t sidx = 0; sidx < T.n_shapes; ++sidx) {
        const float w = sk.bs_w[T.w_off + sidx];
        const uint2 *r = r0 + sidx * shape_stride;
        const uint2 hx = r[0 * 32], hy = r[1 * 32], hz = r[2 * 32], hnx = r[3 * 32], hny = r[4 * 32], hnz = r[5 * 32];
        bs_axpy(x4, hx, w);
        bs_axpy(y4, hy, w);
        bs_axpy(z4, hz, w);
        bs_axpy(nx4, hnx, w);
        bs_axpy(ny4, hny, w);
        bs_axpy(nz4, hnz, w);
    }
}

// BlendShapesContainer's records (9 halfs per vertex and layer: position, normal, tangent) -> the blocked device layout
__global__ void __launch_bounds__(kBlock) k_bs_layout(const uint32_t n_verts, const uint32_t n_shapes, const uint32_t layer_stride,
                                                      const uint16_t *rec, uint16_t *dst, const uint32_t bs_blocks)
{
    const uint64_t t = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
    const uint64_t per_shape = (uint64_t)bs_blocks * 128;
    if (t >= per_shape * n_shapes) return;
    const uint32_t sidx = (uint32_t)(t / per_shape), v = (uint32_t)(t % per_shape);
    uint16_t h[6] = {0, 0, 0, 0, 0, 0};
    if (v < n_verts) {
        const uint16_t *r = rec + ((size_t)sidx * layer_stride + v) * 9;
        for (int k = 0; k < 6; ++k) h[k] = r[k];
    }
    // (shape, block) = 6 rows x 32 groups x 4 halfs
    uint16_t *blk = dst + ((size_t)sidx * bs_blocks + (v >> 7)) * (kBsBlockU2 * 4);
    const uint32_t g = (v >> 2) & 31u, j = v & 3u;
    for (int k = 0; k < 6; ++k) blk[(k * 32 + g) * 4 + j] = h[k];
}

void launch_bs_layout(cudaStream_t s, uint32_t n_verts, uint32_t n_shapes, uint32_t layer_stride, const uint16_t *d_records, uint2 *d_dst, uint32_t bs_blocks)
{
    if (!n_shapes || !bs_blocks) return;
    k_bs_layout<<<(unsigned)(((uint64_t)bs_blocks * 128 * n_shapes + kBlock - 1) / kBlock), kBlock, 0, s>>>(n_verts, n_shapes, layer_stride, d_records,
                                                                                                        reinterpret_cast<uint16_t *>(d_dst), bs_blocks);
}

// The 32 groups of a warp are 128 consecutive vertices, i.e. 1 536 contiguous bytes of each output stream.  Lane l puts its
// three float4 at stage[3l + j] (a quarter-warp's 128-bit stores land in the distinct 16-byte bank groups 3l + j mod 8) and
// the warp reads them back as stage[l + 32j], so each STG.128 writes 512 contiguous bytes: 6 full-line store instructions per
// warp and group instead of 6 that each cover half of 48 sectors.  n_f4 = float4 of the warp's valid groups (3 per group).
__device__ __forceinline__ void store_lines(float4 *stage, const uint32_t lane, const bool valid, const float4 (&p)[3], const float4 (&n)[3],
                                            float4 *po, float4 *no, const uint32_t n_f4)
{
    if (valid) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            stage[3 * lane + j] = p[j];
            stage[96 + 3 * lane + j] = n[j];
        }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const uint32_t i = lane + 32u * j;
        if (i < n_f4) {
            st_stream(po + i, stage[i]);
            st_stream(no + i, stage[96 + i]);
        }
    }
    __syncwarp(); // every lane has read the stage before the next group overwrites it
}

__device__ __forceinline__ void cp_async16(float4 *dst, const float4 *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// a coded group as read from the ring (its 10 float4 and the block's header in iq) -> the raw rows
__device__ __forceinline__ void decode_group(float4 &x4, float4 &y4, float4 &z4, float4 &nx4, float4 &ny4, float4 &nz4, float4 &w0, float4 &w1,
                                             float4 &w2, float4 &w3, uint4 &iq)
{
    float4 *const rows[vcode::kRows] = {&x4, &y4, &z4, &nx4, &ny4, &nz4, &w0, &w1, &w2, &w3};
    uint32_t w[vcode::kWords];
#pragma unroll
    for (int r = 0; r < vcode::kRows; ++r) {
        w[4 * r + 0] = __float_as_uint(rows[r]->x);
        w[4 * r + 1] = __float_as_uint(rows[r]->y);
        w[4 * r + 2] = __float_as_uint(rows[r]->z);
        w[4 * r + 3] = __float_as_uint(rows[r]->w);
    }
    const uint32_t h[3] = {iq.x, iq.y, iq.z};
    float v[vcode::kRows][4];
    uint32_t idx[4];
    vcode::unpack_group(w, h, v, idx);
#pragma unroll
    for (int r = 0; r < vcode::kRows; ++r) *rows[r] = make_float4(v[r][0], v[r][1], v[r][2], v[r][3]);
    iq = make_uint4(idx[0], idx[1], idx[2], idx[3]);
}

constexpr int kSkinStageF4 = 2 * 96;        // per warp: 128 skinned positions + 128 normals
constexpr int kSkinRingF4 = kVblkRows * 32; // per warp: the next group of every lane, 11 rows x 32 lanes (5 632 B)
// shared memory of k_skin: palette planes, output stages, and with PREFETCH the input ring
template <int S, int LOG2C, bool PREFETCH> constexpr size_t skin_smem_bytes()
{
    return sizeof(float4) * ((size_t)3 * S * (1 << LOG2C) + (kBlock / 32) * (kSkinStageF4 + (PREFETCH ? kSkinRingF4 : 0)));
}

// One CTA per tile; a warp skins 32 consecutive groups (128 vertices) per step and writes them as full lines (store_lines).
// PREFETCH: while group i is computed, group i + 1 of the same lane is already on its way into the warp's shared ring by
// 11 cp.async.cg 16-byte copies (a coded block, fyx_vcode.cuh: the group's 10 float4 and the block's header, decoded in
// registers after the reads); lane l only ever reads the 16-byte pieces it copied itself, so cp.async.wait_group is the
// whole synchronisation (no mbarrier, no __syncwarp, no bank conflicts: a row of the ring is 32 consecutive float4).  The
// first copies are issued before griddepcontrol.wait (the vertex blocks are static).  Without PREFETCH the inputs are loaded
// straight into registers (LDG.128, L1-bypassing): the form for palettes too large to leave room for the ring at 2 CTAs/SM.
template <int S, int LOG2C, int MINB, bool BS, bool PREFETCH>
__global__ void __launch_bounds__(kBlock, MINB) k_skin(const SkinArrays sk, const SkinTile *__restrict__ tiles, const uint32_t n_tiles,
                                                     const float one, const float negzero)
{
    constexpr int PAL = 3 * S * (1 << LOG2C);
    extern __shared__ float4 smem[];
    float4 *const s_pal = smem;
    const PackedConsts kc = packed_consts(one, negzero);
    const SkinTile T = tiles[blockIdx.x];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    float4 *const stage = smem + PAL + warp * kSkinStageF4;
    float4 *const ring = smem + PAL + (kBlock / 32) * kSkinStageF4 + warp * kSkinRingF4 + lane; // this lane's column
    const uint32_t zero = __float_as_uint(negzero) << 1; // 0, but not a constant the compiler can fold
    // the lane's block is coded (fyx_vcode.cuh): bit (block - the tile's first block) of the tile
    auto coded_of = [&](const uint32_t q) {
        const uint32_t s = ((T.quad_start + q) >> 5) - (T.quad_start >> 5);
        return (((s < 32 ? T.vcoded[0] : s < 64 ? T.vcoded[1] : T.vcoded[2]) >> (s & 31u)) & 1u) != 0u;
    };
    auto prefetch = [&](const uint32_t q, const uint32_t dep) {
        if (q < T.n_quads) {
            const size_t quad = (size_t)T.quad_start + q;
            const float4 *blk = sk.vblk + (quad >> 5) * kVblkStride, *row = blk + (quad & 31);
#pragma unroll
            for (int r = 0; r < vcode::kRows; ++r) cp_async16(ring + r * 32 + dep, row + r * 32);
            // the 11th copy: the index row of a raw block, the header of a coded one
            cp_async16(ring + 10 * 32 + dep, coded_of(q) ? blk + vcode::kHeaderF4 : row + 10 * 32);
        }
        cp_async_commit();
    };
    if (PREFETCH) prefetch(threadIdx.x, 0);
    pdl_wait(); // the palettes come from k_palette
    skin_fill_palette<S, LOG2C>(s_pal, sk.palette, T.bone_off, T.n_bones);
    __syncthreads();
    for (uint32_t q0 = warp * 32; q0 < T.n_quads; q0 += kBlock) {
        const uint32_t q = q0 + lane;
        const bool valid = q < T.n_quads;
        const size_t quad = (size_t)T.quad_start + q;
        float4 x4, y4, z4, nx4, ny4, nz4, w0, w1, w2, w3;
        uint4 iq;
        if (PREFETCH) {
            cp_async_wait_all();
            if (valid) {
                x4 = ring[0 * 32]; y4 = ring[1 * 32]; z4 = ring[2 * 32];
                nx4 = ring[3 * 32]; ny4 = ring[4 * 32]; nz4 = ring[5 * 32];
                w0 = ring[6 * 32]; w1 = ring[7 * 32]; w2 = ring[8 * 32]; w3 = ring[9 * 32];
                iq = *reinterpret_cast<const uint4 *>(ring + 10 * 32);
            }
            // the next copies overwrite the slots just read: their address depends on a value of every one of those 11 reads,
            // so no copy can be issued before the reads have completed
            const uint32_t dep = valid ? ((__float_as_uint(x4.x) ^ __float_as_uint(y4.x) ^ __float_as_uint(z4.x) ^ __float_as_uint(nx4.x) ^
                                           __float_as_uint(ny4.x) ^ __float_as_uint(nz4.x) ^ __float_as_uint(w0.x) ^ __float_as_uint(w1.x) ^
                                           __float_as_uint(w2.x) ^ __float_as_uint(w3.x) ^ iq.x) & zero)
                                       : 0u;
            if (valid && coded_of(q)) decode_group(x4, y4, z4, nx4, ny4, nz4, w0, w1, w2, w3, iq);
            prefetch(q + kBlock, dep);
        } else if (valid) {
            const float4 *row = sk.vblk + (quad >> 5) * kVblkStride + (quad & 31); // block, then this group's column
            x4 = ld_stream(row + 0 * 32); y4 = ld_stream(row + 1 * 32); z4 = ld_stream(row + 2 * 32);
            nx4 = ld_stream(row + 3 * 32); ny4 = ld_stream(row + 4 * 32); nz4 = ld_stream(row + 5 * 32);
            w0 = ld_stream(row + 6 * 32); w1 = ld_stream(row + 7 * 32); w2 = ld_stream(row + 8 * 32); w3 = ld_stream(row + 9 * 32);
            iq = ld_stream(reinterpret_cast<const uint4 *>(row + 10 * 32));
        }
        float4 p[3], n[3];
        if (valid) {
            if (BS && T.n_shapes) apply_blend_shapes(sk, T, q, x4, y4, z4, nx4, ny4, nz4);
            skin_quad_regs<S, LOG2C>(s_pal, lane, x4, y4, z4, nx4, ny4, nz4, w0, w1, w2, w3, iq, p, n, kc);
        }
        const size_t f0 = 3 * ((size_t)T.quad_start + q0); // the warp's first float4 in each output stream
        store_lines(stage, lane, valid, p, n, reinterpret_cast<float4 *>(sk.opos) + f0, reinterpret_cast<float4 *>(sk.onrm) + f0,
                    3u * min(32u, T.n_quads - q0));
    }
}

// ------------------------------------------------------------------------------------------------
// Host-facing scatter / gather between the caller's AoS-by-node-index arrays and the slot-ordered
// SoA planes.  Invalid indices are skipped (Pool::try_borrow semantics).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t resolve_slot(const uint32_t *d_idx, uint32_t e, const uint32_t *slot_of_node,
                                                 uint32_t n_nodes)
{
    const uint32_t node = d_idx ? d_idx[e] : e;
    if (node >= n_nodes) return FYX_NONE;
    return slot_of_node[node];
}

// bottom row must be bit-exactly (+0,+0,+0,1) — what Transform::calculate_local_transform writes
// (scene/transform.rs:479-536) — and all entries finite; returns false otherwise
__device__ __forceinline__ bool load_affine_rows(const float *m16, Affine &A)
{
    const float4 *c = reinterpret_cast<const float4 *>(m16);
    const float4 c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3];
    A.r0 = make_float4(c0.x, c1.x, c2.x, c3.x);
    A.r1 = make_float4(c0.y, c1.y, c2.y, c3.y);
    A.r2 = make_float4(c0.z, c1.z, c2.z, c3.z);
    const bool bottom = (__float_as_uint(c0.w) == 0u) & (__float_as_uint(c1.w) == 0u) & (__float_as_uint(c2.w) == 0u) &
                        (c3.w == 1.0f);
    return bottom & finite4(A.r0) & finite4(A.r1) & finite4(A.r2);
}

__global__ void __launch_bounds__(kBlock) k_scatter_locals(const NodeArrays a, const uint32_t count, const uint32_t *d_idx,
                                                           const float *d_m16, const uint32_t *slot_of_node,
                                                           const uint32_t n_nodes, uint32_t *d_err)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    if (slot == FYX_NONE) return;
    Affine A;
    if (!load_affine_rows(d_m16 + 16 * (size_t)e, A)) {
        atomicOr(d_err, E_NOT_AFFINE);
        return;
    }
    a.L[0][slot] = A.r0;
    a.L[1][slot] = A.r1;
    a.L[2][slot] = A.r2;
    atomicOr(a.flags + slot, F_DIRTY_SELF); // NodeMessageKind::TransformChanged
}

// Transform::calculate_local_transform (scene/transform.rs:421-540), expression by expression (Rust's
// a + b - c ... is left-associative; x - y is x + (-y)).  One thread per changed node.
// ROT_ONLY: the payload is just the new rotation (16 B); position and scale come from the device-resident copy of
// the node's last full record (trs_by_slot), which every call keeps up to date — property-level change tracking:
// skeletal animation mostly rewrites rotations (Transform::set_rotation), so 20 B per bone cross PCIe instead of 44.
template <bool HAS_STATICS, bool ROT_ONLY>
__global__ void __launch_bounds__(kBlock) k_scatter_trs(const NodeArrays a, const uint32_t count, const uint32_t *d_idx,
                                                        const void *d_payload, fyx_trs *trs_by_slot,
                                                        const fyx_transform_statics *st_by_slot, const uint32_t *slot_of_node,
                                                        const uint32_t n_nodes, uint32_t *d_err)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    if (slot == FYX_NONE) return;
    fyx_trs t;
    if (ROT_ONLY) {
        t = trs_by_slot[slot];
        const float4 q = static_cast<const float4 *>(d_payload)[e];
        t.rotation[0] = q.x; t.rotation[1] = q.y; t.rotation[2] = q.z; t.rotation[3] = q.w;
    } else {
        t = static_cast<const fyx_trs *>(d_payload)[e];
    }
    if (trs_by_slot) trs_by_slot[slot] = t;
    Affine A;
    trs_to_local<HAS_STATICS>(t, HAS_STATICS ? st_by_slot + slot : nullptr, A);
    if (!(finite4(A.r0) & finite4(A.r1) & finite4(A.r2))) {
        atomicOr(d_err, E_NOT_AFFINE);
        return;
    }
    a.L[0][slot] = A.r0;
    a.L[1][slot] = A.r1;
    a.L[2][slot] = A.r2;
    atomicOr(a.flags + slot, F_DIRTY_SELF); // NodeMessageKind::TransformChanged
}

// one thread per word of the records
__global__ void __launch_bounds__(kBlock) k_scatter_words(uint32_t *dst, const uint32_t words, const uint32_t count,
                                                          const uint32_t *d_idx, const uint32_t *d_val,
                                                          const uint32_t *slot_of_node, const uint32_t n_nodes)
{
    const uint64_t t = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
    if (t >= (uint64_t)count * words) return;
    const uint32_t e = (uint32_t)(t / words), w = (uint32_t)(t % words);
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    if (slot == FYX_NONE) return;
    dst[(size_t)slot * words + w] = d_val[t];
}

__global__ void __launch_bounds__(kBlock) k_scatter_flags(uint32_t *flags, const uint32_t count, const uint32_t *d_idx,
                                                          const uint32_t *d_val, const uint32_t *slot_of_node,
                                                          const uint32_t n_nodes)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    if (slot == FYX_NONE) return;
    constexpr uint32_t settable = FYX_NODE_INPUT_MASK & ~FYX_NODE_ALIVE;
    flags[slot] = (flags[slot] & ~settable) | (d_val[e] & settable);
}

__global__ void __launch_bounds__(kBlock) k_scatter_aabbs(const NodeArrays a, const uint32_t count, const uint32_t *d_idx,
                                                          const float *d_aabb6, const uint32_t *slot_of_node,
                                                          const uint32_t n_nodes)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    if (slot == FYX_NONE) return;
    const float *b = d_aabb6 + 6 * (size_t)e;
    a.la[0][slot] = make_float2(b[0], b[3]);
    a.la[1][slot] = make_float2(b[1], b[4]);
    a.la[2][slot] = make_float2(b[2], b[5]);
    atomicOr(a.flags + slot, F_DIRTY_SELF); // world box must be rebuilt
}

__global__ void __launch_bounds__(kBlock) k_gather_globals(const NodeArrays a, const uint32_t count, const uint32_t *d_idx,
                                                           const uint32_t *slot_of_node, const uint32_t n_nodes,
                                                           float *d_out)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    Affine Gm = affine_identity();
    if (slot != FYX_NONE) {
        Gm.r0 = a.G[0][slot];
        Gm.r1 = a.G[1][slot];
        Gm.r2 = a.G[2][slot];
    }
    float4 *o = reinterpret_cast<float4 *>(d_out + 16 * (size_t)e);
    o[0] = make_float4(Gm.r0.x, Gm.r1.x, Gm.r2.x, 0.0f);
    o[1] = make_float4(Gm.r0.y, Gm.r1.y, Gm.r2.y, 0.0f);
    o[2] = make_float4(Gm.r0.z, Gm.r1.z, Gm.r2.z, 0.0f);
    o[3] = make_float4(Gm.r0.w, Gm.r1.w, Gm.r2.w, 1.0f);
}

__global__ void __launch_bounds__(kBlock) k_gather_aabbs(const NodeArrays a, const uint32_t count, const uint32_t *d_idx,
                                                         const uint32_t *slot_of_node, const uint32_t n_nodes, float *d_out)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    float *o = d_out + 6 * (size_t)e;
    if (slot == FYX_NONE) { // AxisAlignedBoundingBox::default()
        o[0] = o[1] = o[2] = 3.402823466e38f;
        o[3] = o[4] = o[5] = -3.402823466e38f;
        return;
    }
    const float2 x = a.wa[0][slot], y = a.wa[1][slot], z = a.wa[2][slot];
    o[0] = x.x; o[1] = y.x; o[2] = z.x;
    o[3] = x.y; o[4] = y.y; o[5] = z.y;
}

__global__ void __launch_bounds__(kBlock) k_gather_flags(const NodeArrays a, const uint32_t count, const uint32_t *d_idx,
                                                         const uint32_t *slot_of_node, const uint32_t n_nodes,
                                                         uint32_t *d_out)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= count) return;
    const uint32_t slot = resolve_slot(d_idx, e, slot_of_node, n_nodes);
    d_out[e] = (slot == FYX_NONE) ? 0u
                                  : (a.flags[slot] & (FYX_NODE_INPUT_MASK | FYX_NODE_GLOBAL_VISIBILITY |
                                                      FYX_NODE_GLOBAL_ENABLED | FYX_NODE_REACHABLE));
}

// VertexBuffer bytes (scene/mesh/buffer.rs:404-414) → the blocked input layout of k_skin (fyx_internal.h).
// Done once per surface at load.  Vertex v (absolute) = group Q = v/4, element j = v%4 of block Q/32.
__global__ void __launch_bounds__(kBlock) k_deinterleave(const uint32_t n_verts, const uint32_t n_padded,
                                                         const unsigned char *d_bytes, const fyx_vertex_layout l,
                                                         const uint32_t n_bones, float4 *vblk, const uint64_t first_vertex,
                                                         uint32_t *d_err)
{
    const uint32_t v = blockIdx.x * kBlock + threadIdx.x;
    if (v >= n_padded) return;
    float p[3] = {0.f, 0.f, 0.f}, n[3] = {0.f, 0.f, 0.f};
    float w[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t bi = 0u;
    if (v < n_verts) {
        const unsigned char *vp = d_bytes + (size_t)v * l.stride;
        const float *fp = reinterpret_cast<const float *>(vp + l.position_offset);
        const float *fn = reinterpret_cast<const float *>(vp + l.normal_offset);
        const float *fw = reinterpret_cast<const float *>(vp + l.bone_weights_offset);
        p[0] = fp[0]; p[1] = fp[1]; p[2] = fp[2];
        n[0] = fn[0]; n[1] = fn[1]; n[2] = fn[2];
        w[0] = fw[0]; w[1] = fw[1]; w[2] = fw[2]; w[3] = fw[3];
        bi = *reinterpret_cast<const uint32_t *>(vp + l.bone_indices_offset);
        uint32_t bad = 0u;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (((bi >> (8 * k)) & 0xFFu) >= n_bones) bad = 1u;
        if (bad) { // the reference would panic on the out-of-range index (mesh/mod.rs:515)
            atomicOr(d_err, E_BAD_BONE_INDEX);
            bi = 0u;
            w[0] = w[1] = w[2] = w[3] = 0.f;
        }
        if (!((fabsf(p[0]) <= 3.402823466e38f) & (fabsf(p[1]) <= 3.402823466e38f) & (fabsf(p[2]) <= 3.402823466e38f)))
            atomicOr(d_err, E_NONFINITE_VERTEX);
    }
    const uint64_t av = first_vertex + v;
    const uint64_t Q = av >> 2;
    const uint32_t j = (uint32_t)(av & 3);
    float *blk = reinterpret_cast<float *>(vblk + (Q >> 5) * kVblkStride + (Q & 31)); // row 0, this group's float4
    const size_t rs = 32 * 4; // floats between rows
    blk[0 * rs + j] = p[0]; blk[1 * rs + j] = p[1]; blk[2 * rs + j] = p[2];
    blk[3 * rs + j] = n[0]; blk[4 * rs + j] = n[1]; blk[5 * rs + j] = n[2];
    blk[6 * rs + j] = w[0]; blk[7 * rs + j] = w[1]; blk[8 * rs + j] = w[2]; blk[9 * rs + j] = w[3];
    reinterpret_cast<uint32_t *>(blk)[10 * rs + j] = bi;
}

// The encode pass of a surface's load (fyx_vcode.cuh): one warp per block the load completes, coded in place where it fits.
__global__ void __launch_bounds__(kBlock) k_vcode(float4 *vblk, uint8_t *vflag, const vcode::LoadBlocks lb)
{
    const uint64_t b = lb.first + (uint64_t)blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
    const uint32_t lane = threadIdx.x & 31u;
    if (b >= lb.complete_end || vflag[b] != vcode::kVflagRaw) return;
    if (vcode::encode_block_warp(reinterpret_cast<uint32_t *>(vblk + b * kVblkStride), lane) && lane == 0) vflag[b] = vcode::kVflagCoded;
}

// every coded block of [0, n_blocks) back to the raw layout, in place: one warp per block
__global__ void __launch_bounds__(kBlock) k_vdecode_all(float4 *vblk, uint8_t *vflag, const uint64_t n_blocks)
{
    const uint64_t b = (uint64_t)blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
    const uint32_t lane = threadIdx.x & 31u;
    if (b >= n_blocks || vflag[b] != vcode::kVflagCoded) return;
    uint32_t *blk = reinterpret_cast<uint32_t *>(vblk + b * kVblkStride);
    uint32_t raw[vcode::kRawF4 * 4 / vcode::kGroups]; // this group's 11 raw float4, gathered before any lane writes
    const uint32_t h[3] = {blk[vcode::kHeaderF4 * 4], blk[vcode::kHeaderF4 * 4 + 1], blk[vcode::kHeaderF4 * 4 + 2]};
    uint32_t w[vcode::kWords], idx[4];
    float v[vcode::kRows][4];
#pragma unroll
    for (int r = 0; r < vcode::kRows; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) w[4 * r + c] = blk[(r * 32 + lane) * 4 + c];
    vcode::unpack_group(w, h, v, idx);
#pragma unroll
    for (int r = 0; r < vcode::kRows; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) raw[4 * r + j] = __float_as_uint(v[r][j]);
#pragma unroll
    for (int j = 0; j < 4; ++j) raw[40 + j] = idx[j];
    __syncwarp(); // the header and every group are read before the raw rows overwrite them
#pragma unroll
    for (int r = 0; r < 11; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) blk[(r * 32 + lane) * 4 + j] = raw[4 * r + j];
    if (lane == 0) vflag[b] = vcode::kVflagRaw;
}

// tile t's bit s: block (quad_start / 32) + s of the tile is coded
__global__ void __launch_bounds__(kBlock) k_tile_vcode(SkinTile *tiles, const uint32_t n_tiles, const uint8_t *vflag)
{
    const uint32_t t = blockIdx.x * kBlock + threadIdx.x;
    if (t >= n_tiles) return;
    SkinTile &T = tiles[t];
    const uint32_t b0 = T.quad_start >> 5, nb = ((T.quad_start + T.n_quads - 1) >> 5) - b0 + 1;
    uint32_t m[3] = {0u, 0u, 0u};
    for (uint32_t s = 0; s < nb; ++s)
        if (vflag[b0 + s] == vcode::kVflagCoded) m[s >> 5] |= 1u << (s & 31);
    for (int k = 0; k < 3; ++k) T.vcoded[k] = m[k];
}

__global__ void __launch_bounds__(kBlock) k_ib_rows(const uint32_t n, const float *d_m16, float4 *r0, float4 *r1, float4 *r2,
                                                    uint32_t *d_err)
{
    const uint32_t e = blockIdx.x * kBlock + threadIdx.x;
    if (e >= n) return;
    Affine A;
    if (!load_affine_rows(d_m16 + 16 * (size_t)e, A)) {
        atomicOr(d_err, E_NOT_AFFINE);
        A = affine_identity();
    }
    r0[e] = A.r0;
    r1[e] = A.r1;
    r2[e] = A.r2;
}

__global__ void k_or_u32(uint32_t *p, const uint32_t bits) { atomicOr(p, bits); }

__global__ void __launch_bounds__(kBlock) k_permute_words(uint32_t *dst, const uint32_t *src, const uint32_t *map, const uint32_t n,
                                                          const WordRecord def)
{
    const uint32_t words = def.words;
    const uint64_t t = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
    if (t >= (uint64_t)n * words) return;
    const uint32_t s = (uint32_t)(t / words), w = (uint32_t)(t % words);
    const uint32_t o = map ? map[s] : FYX_NONE;
    dst[t] = (o != FYX_NONE) ? src[(size_t)o * words + w] : def.w[w];
}

// After the fixed-slot NCCL all-gather of a visible list: rank r's entries sit at pad[r*maxc ..];
// pack them back to back (rank order) so every rank holds one contiguous list per frustum.
__global__ void __launch_bounds__(kBlock) k_compact_gathered(const uint32_t *pad, const uint32_t maxc,
                                                             const uint32_t *counts_all, const int nranks, const int f,
                                                             uint32_t *dst)
{
    const uint64_t i = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
    if (!maxc) return;
    const uint32_t r = (uint32_t)(i / maxc), j = (uint32_t)(i % maxc);
    if (r >= (uint32_t)nranks) return;
    if (j >= counts_all[r * FYX_MAX_FRUSTA + f]) return;
    uint32_t off = 0;
    for (uint32_t q = 0; q < r; ++q) off += counts_all[q * FYX_MAX_FRUSTA + f];
    dst[off + j] = pad[(size_t)r * maxc + j];
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
static inline unsigned grid_for(uint64_t n) { return (unsigned)((n + kBlock - 1) / kBlock); }

// The usual frustum counts get an unrolled cull: camera, CSM cascades, cube faces.
template <int NFT>
static void launch_update_level_t(cudaStream_t s, const NodeArrays &a, uint32_t lo, uint32_t hi, bool update_all, const CullParams &cp)
{
    if (update_all) launch_pdl(k_update_level<NFT, true>, grid_for(hi - lo), kBlock, 0, s, a, lo, hi, 1u, cp);
    else launch_pdl(k_update_level<NFT, false>, grid_for(hi - lo), kBlock, 0, s, a, lo, hi, 0u, cp);
}

void launch_update_level(cudaStream_t s, const NodeArrays &a, uint32_t lo, uint32_t hi, bool update_all, const CullParams *cull)
{
    if (hi <= lo) return;
    if (!cull) {
        CullParams none;
        none.nf = 0;
        launch_update_level_t<-1>(s, a, lo, hi, update_all, none);
        return;
    }
    switch (cull->nf) {
    case 1: launch_update_level_t<1>(s, a, lo, hi, update_all, *cull); break;
    case 2: launch_update_level_t<2>(s, a, lo, hi, update_all, *cull); break;
    case 3: launch_update_level_t<3>(s, a, lo, hi, update_all, *cull); break;
    case 4: launch_update_level_t<4>(s, a, lo, hi, update_all, *cull); break;
    case 6: launch_update_level_t<6>(s, a, lo, hi, update_all, *cull); break;
    default: launch_update_level_t<0>(s, a, lo, hi, update_all, *cull); break;
    }
}

template <int NFT> static void launch_subforest_t(cudaStream_t s, const NodeArrays &a, const SubforestPlan &sf, bool ua, const CullParams &cp)
{
    if (ua) launch_pdl(k_update_subforest<NFT, true>, sf.n_ctas, kBlock, 0, s, a, sf.rng, (int)sf.n_levels, 1u, cp);
    else launch_pdl(k_update_subforest<NFT, false>, sf.n_ctas, kBlock, 0, s, a, sf.rng, (int)sf.n_levels, 0u, cp);
}

void launch_update_subforest(cudaStream_t s, const NodeArrays &a, const SubforestPlan &sf, bool update_all, const CullParams *cull)
{
    if (!sf.n_ctas || !sf.n_levels) return;
    if (!cull) {
        CullParams none;
        none.nf = 0;
        launch_subforest_t<-1>(s, a, sf, update_all, none);
        return;
    }
    switch (cull->nf) {
    case 1: launch_subforest_t<1>(s, a, sf, update_all, *cull); break;
    case 6: launch_subforest_t<6>(s, a, sf, update_all, *cull); break;
    default: launch_subforest_t<0>(s, a, sf, update_all, *cull); break;
    }
}

// Reflection-probe selection of from_graph (renderer/bundle.rs:918-925): the last ReflectionProbe in pool order whose world box
// contains the observer (AxisAlignedBoundingBox::is_contains_point, inclusive) — atomicMax over (node index + 1) per observer.
__global__ void __launch_bounds__(kBlock) k_select_probes(const NodeArrays a, const Observers obs, uint32_t *best)
{
    const uint32_t slot = blockIdx.x * kBlock + threadIdx.x;
    if (slot >= a.cap) return;
    const uint32_t nf = a.flags[slot];
    if ((nf & (FYX_NODE_ALIVE | FYX_NODE_REFLECTION_PROBE)) != (FYX_NODE_ALIVE | FYX_NODE_REFLECTION_PROBE)) return;
    const float2 wx = a.wa[0][slot], wy = a.wa[1][slot], wz = a.wa[2][slot];
    const uint32_t gi = a.gidx[slot];
    for (uint32_t f = 0; f < obs.n; ++f) {
        const float px = obs.o[f].translation[0], py = obs.o[f].translation[1], pz = obs.o[f].translation[2];
        if (px >= wx.x && px <= wx.y && py >= wy.x && py <= wy.y && pz >= wz.x && pz <= wz.y) atomicMax(best + f, gi + 1u);
    }
}

void launch_select_probes(cudaStream_t s, const NodeArrays &a, const Observers &obs, uint32_t *best)
{
    if (!a.cap || !obs.n) return;
    k_select_probes<<<grid_for(a.cap), kBlock, 0, s>>>(a, obs, best);
}

void launch_cull_lights(cudaStream_t s, const NodeArrays &a, const CullParams &cp, uint32_t *const *d_out_ptrs, uint32_t *counts)
{
    if (!a.cap) return;
    k_cull_lights<<<grid_for(a.cap), kBlock, 0, s>>>(a, cp, d_out_ptrs, counts);
}

uint32_t launch_cull(cudaStream_t s, const NodeArrays &a, const CullParams &cp, const MapParams::Prune &pr, const Observers &obs,
                     const uint32_t *pr_level_off, uint32_t n_levels)
{
    uint32_t n = 0u;
    for (uint32_t l = 0; l < n_levels; ++l) {
        const uint32_t lo = pr_level_off[l], hi = pr_level_off[l + 1];
        if (hi <= lo) continue;
        k_cull_pruners<<<grid_for(hi - lo), kBlock, 0, s>>>(a, cp, pr, obs, lo, hi);
        ++n;
    }
    if (!a.cap) return n;
    const unsigned g = grid_for(a.cap);
    switch (cp.nf) {
    case 1: k_cull<1><<<g, kBlock, 0, s>>>(a, cp, pr); break;
    case 2: k_cull<2><<<g, kBlock, 0, s>>>(a, cp, pr); break;
    case 3: k_cull<3><<<g, kBlock, 0, s>>>(a, cp, pr); break;
    case 4: k_cull<4><<<g, kBlock, 0, s>>>(a, cp, pr); break;
    case 6: k_cull<6><<<g, kBlock, 0, s>>>(a, cp, pr); break;
    default: k_cull<0><<<g, kBlock, 0, s>>>(a, cp, pr); break;
    }
    return n + 1u;
}

void launch_fold_bones(cudaStream_t s, const NodeArrays &a, const FoldArrays &fa, const CullParams *cull)
{
    if (!fa.n) return;
    const unsigned grid = grid_for((uint64_t)fa.n * 32); // one warp per skinned mesh
    if (cull) {
        switch (cull->nf) {
        case 1: launch_pdl(k_fold_bones<1>, grid, kBlock, 0, s, a, fa, *cull); break;
        case 6: launch_pdl(k_fold_bones<6>, grid, kBlock, 0, s, a, fa, *cull); break;
        default: launch_pdl(k_fold_bones<0>, grid, kBlock, 0, s, a, fa, *cull); break;
        }
    } else {
        CullParams none;
        none.nf = 0;
        launch_pdl(k_fold_bones<-1>, grid, kBlock, 0, s, a, fa, none);
    }
}

void launch_snapshot_bones(cudaStream_t s, const NodeArrays &a, uint32_t n_late, const uint32_t *late_slot, float4 *stale_pos)
{
    if (!n_late) return;
    k_snapshot_bones<<<grid_for(n_late), kBlock, 0, s>>>(a, n_late, late_slot, stale_pos);
}

void launch_palette(cudaStream_t s, const NodeArrays &a, const SkinArrays &sk)
{
    if (!sk.n_entries) return;
    launch_pdl(k_palette, grid_for(sk.n_entries), kBlock, 0, s, a, sk);
}

template <int S, int LOG2C, int MINB, bool BS, bool PREFETCH>
static void launch_skin_t2(cudaStream_t s, const SkinArrays &sk, const SkinTile *tiles, uint32_t n_tiles)
{
    constexpr size_t smem = skin_smem_bytes<S, LOG2C, PREFETCH>();
    static bool init = false;
    if (!init) {
        cudaFuncSetAttribute(k_skin<S, LOG2C, MINB, BS, PREFETCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        init = true;
    }
    launch_pdl(k_skin<S, LOG2C, MINB, BS, PREFETCH>, n_tiles, kBlock, smem, s, sk, tiles, n_tiles, 1.0f, -0.0f);
}
template <int S, int LOG2C, int MINB, bool PREFETCH>
static void launch_skin_t(cudaStream_t s, const SkinArrays &sk, const SkinTile *tiles, uint32_t n_tiles, bool bs)
{
    if (bs) launch_skin_t2<S, LOG2C, MINB, true, PREFETCH>(s, sk, tiles, n_tiles);
    else launch_skin_t2<S, LOG2C, MINB, false, PREFETCH>(s, sk, tiles, n_tiles);
}

void launch_skin(cudaStream_t s, const SkinArrays &sk, const SkinTile *tiles, uint32_t n_tiles, uint32_t max_bones, bool blend_shapes)
{
    if (!n_tiles) return;
    // <= 64 bones: the prefetching form, 2 CTAs/SM (<= 128 registers; 25 KB palette + 24 KB output stages + 44 KB ring per CTA).
    // Larger palettes leave no room for the ring at 2 CTAs/SM: loads into registers, 3 CTAs/SM (<= 85 registers).
    static_assert(kSkinRingMaxBones == 64, "the prefetching form (the one that reads coded blocks) holds 65 palette entries");
    if (max_bones <= 64) {       // 8 copies: 25 KB of palette planes
        launch_skin_t<65, 3, 2, true>(s, sk, tiles, n_tiles, blend_shapes);
    } else if (max_bones <= 128) { // 8 copies: 50 KB
        launch_skin_t<129, 3, 3, false>(s, sk, tiles, n_tiles, blend_shapes);
    } else {                       // 4 copies (2-way worst case): 49 KB
        launch_skin_t<257, 2, 3, false>(s, sk, tiles, n_tiles, blend_shapes);
    }
}

void launch_scatter_locals(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx, const float *d_m16,
                           const uint32_t *slot_of_node, uint32_t n_nodes, uint32_t *d_err)
{
    if (!count) return;
    k_scatter_locals<<<grid_for(count), kBlock, 0, s>>>(a, count, d_idx, d_m16, slot_of_node, n_nodes, d_err);
}

void launch_scatter_trs(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx, const void *d_payload, bool rot_only,
                        fyx_trs *trs_by_slot, const fyx_transform_statics *st, const uint32_t *slot_of_node, uint32_t n_nodes,
                        uint32_t *d_err)
{
    if (!count) return;
    const unsigned g = grid_for(count);
    if (rot_only) {
        if (st) k_scatter_trs<true, true><<<g, kBlock, 0, s>>>(a, count, d_idx, d_payload, trs_by_slot, st, slot_of_node, n_nodes, d_err);
        else k_scatter_trs<false, true><<<g, kBlock, 0, s>>>(a, count, d_idx, d_payload, trs_by_slot, st, slot_of_node, n_nodes, d_err);
    } else {
        if (st) k_scatter_trs<true, false><<<g, kBlock, 0, s>>>(a, count, d_idx, d_payload, trs_by_slot, st, slot_of_node, n_nodes, d_err);
        else k_scatter_trs<false, false><<<g, kBlock, 0, s>>>(a, count, d_idx, d_payload, trs_by_slot, st, slot_of_node, n_nodes, d_err);
    }
}

void launch_scatter_words(cudaStream_t s, uint32_t *dst, uint32_t words, uint32_t count, const uint32_t *d_idx,
                          const uint32_t *d_val, const uint32_t *slot_of_node, uint32_t n_nodes)
{
    if (!count || !words) return;
    k_scatter_words<<<grid_for((uint64_t)count * words), kBlock, 0, s>>>(dst, words, count, d_idx, d_val, slot_of_node, n_nodes);
}

void launch_scatter_flags(cudaStream_t s, uint32_t *flags, uint32_t count, const uint32_t *d_idx,
                          const uint32_t *d_val, const uint32_t *slot_of_node, uint32_t n_nodes)
{
    if (!count) return;
    k_scatter_flags<<<grid_for(count), kBlock, 0, s>>>(flags, count, d_idx, d_val, slot_of_node, n_nodes);
}

void launch_scatter_aabbs(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx, const float *d_aabb6,
                          const uint32_t *slot_of_node, uint32_t n_nodes)
{
    if (!count) return;
    k_scatter_aabbs<<<grid_for(count), kBlock, 0, s>>>(a, count, d_idx, d_aabb6, slot_of_node, n_nodes);
}

void launch_gather_globals(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                           const uint32_t *slot_of_node, uint32_t n_nodes, float *d_out)
{
    if (!count) return;
    k_gather_globals<<<grid_for(count), kBlock, 0, s>>>(a, count, d_idx, slot_of_node, n_nodes, d_out);
}

void launch_gather_aabbs(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                         const uint32_t *slot_of_node, uint32_t n_nodes, float *d_out6)
{
    if (!count) return;
    k_gather_aabbs<<<grid_for(count), kBlock, 0, s>>>(a, count, d_idx, slot_of_node, n_nodes, d_out6);
}

void launch_gather_flags(cudaStream_t s, const NodeArrays &a, uint32_t count, const uint32_t *d_idx,
                         const uint32_t *slot_of_node, uint32_t n_nodes, uint32_t *d_out)
{
    if (!count) return;
    k_gather_flags<<<grid_for(count), kBlock, 0, s>>>(a, count, d_idx, slot_of_node, n_nodes, d_out);
}

void launch_deinterleave(cudaStream_t s, uint32_t n_verts, const unsigned char *d_bytes, fyx_vertex_layout layout,
                         uint32_t n_bones, float4 *vblk, uint8_t *vflag, bool code, uint64_t first_vertex, uint32_t *d_err)
{
    const uint32_t n_padded = (n_verts + 3u) & ~3u;
    if (!n_padded) return;
    k_deinterleave<<<grid_for(n_padded), kBlock, 0, s>>>(n_verts, n_padded, d_bytes, layout, n_bones, vblk, first_vertex, d_err);
    const vcode::LoadBlocks lb = vcode::load_blocks(first_vertex, n_padded);
    if (code && lb.complete_end > lb.first) k_vcode<<<grid_for((lb.complete_end - lb.first) * 32), kBlock, 0, s>>>(vblk, vflag, lb);
}

void launch_vdecode_all(cudaStream_t s, float4 *vblk, uint8_t *vflag, uint64_t n_blocks)
{
    if (n_blocks) k_vdecode_all<<<grid_for(n_blocks * 32), kBlock, 0, s>>>(vblk, vflag, n_blocks);
}

void launch_tile_vcode(cudaStream_t s, SkinTile *tiles, uint32_t n_tiles, const uint8_t *vflag)
{
    if (n_tiles) k_tile_vcode<<<grid_for(n_tiles), kBlock, 0, s>>>(tiles, n_tiles, vflag);
}

void launch_ib_rows(cudaStream_t s, uint32_t n, const float *d_m16, float4 *r0, float4 *r1, float4 *r2, uint32_t *d_err)
{
    if (!n) return;
    k_ib_rows<<<grid_for(n), kBlock, 0, s>>>(n, d_m16, r0, r1, r2, d_err);
}

void launch_or_u32(cudaStream_t s, uint32_t *p, uint32_t bits) { k_or_u32<<<1, 1, 0, s>>>(p, bits); }

void launch_permute_words(cudaStream_t s, void *dst, const void *src, const uint32_t *map, uint32_t n, const WordRecord &def)
{
    if (!n || !def.words) return;
    k_permute_words<<<grid_for((uint64_t)n * def.words), kBlock, 0, s>>>(static_cast<uint32_t *>(dst), static_cast<const uint32_t *>(src), map, n, def);
}

void launch_compact_gathered(cudaStream_t s, const uint32_t *pad, uint32_t maxc, const uint32_t *counts_all, int nranks, int f,
                             uint32_t *dst)
{
    if (!maxc || nranks <= 0) return;
    k_compact_gathered<<<grid_for((uint64_t)maxc * nranks), kBlock, 0, s>>>(pad, maxc, counts_all, nranks, f, dst);
}

// ------------------------------------------------------------------------------------------------
// N4 shadow casters (fyx_cull_shadow_casters[_csm]): the shadow-map loop of the deferred light renderer (renderer/light.rs:509-606,
// 695-782) and, for every map, the cull of RenderDataBundleStorage::from_graph in its shadow pass (renderer/shadow/spot.rs:142,
// shadow/point.rs:162-180, shadow/csm.rs:251-265).  Pass 1 (one CTA) builds the map table: 1 map per spot light, 6 per
// point light, 3 cascades per directional light; pass 2 reads every node once and counts its entries in
// every map; a one-CTA scan places the lists; pass 3 re-tests the warps that had an entry and writes the lists.
// The passes after the table are those of every many-map cull (MapParams): the observers and their shadow maps bring
// their own table kernel and a form of the node passes' predicate.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kShadowNeed = kNeedBits | FYX_NODE_CAST_SHADOWS;

// The ordered scan of a one-CTA kernel of BLOCK threads, in shared memory.  excl: every thread gives v and gets the sum of
// the v of the threads before it (plus *from, read after the barrier), so what the threads place at their offsets keeps
// thread order.  place: the same over rounds, offsets counted from `base`, which it carries from round to round: thread 0
// clears it before the first round, with no barrier of its own, because `base` is only ever read after excl's barrier;
// after the last round it is the sum of all.  A kernel that carries bases of its own (k_scene_shadow_maps) uses excl
// alone and leaves `base` unused.
template <uint32_t BLOCK> struct BlockScan {
    uint32_t warp[BLOCK / 32u];
    uint32_t base;
    __device__ __forceinline__ uint32_t excl(const uint32_t v, const uint32_t *from = nullptr)
    {
        const uint32_t lane = threadIdx.x & 31u, w_self = threadIdx.x >> 5;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= (uint32_t)o) incl += t;
        }
        if (lane == 31u) warp[w_self] = incl;
        __syncthreads();
        uint32_t e = from ? *from + incl - v : incl - v;
        for (uint32_t w = 0; w < w_self; ++w) e += warp[w];
        return e;
    }
    __device__ __forceinline__ uint32_t place(const uint32_t v)
    {
        const uint32_t first = excl(v, &base);
        __syncthreads();
        if (threadIdx.x == BLOCK - 1u) base = first + v;
        __syncthreads();
        return first;
    }
};

// Vector3::try_normalize(f32::EPSILON).unwrap_or(fallback): norm <= eps ⇒ the fallback, else each component / norm
__device__ __forceinline__ void try_normalize(const float *v, const float *fallback, float *out)
{
    const float n = sqrtf(dot3(v, v));
    if (n <= 1.1920929e-07f) {
        out[0] = fallback[0]; out[1] = fallback[1]; out[2] = fallback[2];
    } else {
        out[0] = v[0] / n; out[1] = v[1] / n; out[2] = v[2] / n;
    }
}

// renderer/utils.rs:49-75, CubeMapFaceDescriptor::cube_faces(): look and up of the six faces
__constant__ float c_face_look[6][3] = {{1.f, 0.f, 0.f}, {-1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, -1.f, 0.f}, {0.f, 0.f, 1.f}, {0.f, 0.f, -1.f}};
__constant__ float c_face_up[6][3] = {{0.f, -1.f, 0.f}, {0.f, -1.f, 0.f}, {0.f, 0.f, 1.f}, {0.f, 0.f, -1.f}, {0.f, -1.f, 0.f}, {0.f, -1.f, 0.f}};

// one map: view_projection = P · V, its frustum (Frustum::default if the matrix has none, renderer/bundle.rs:893-896) with
// the render mask of the observer that renders it
__device__ __forceinline__ void shadow_map_out(const MapParams &mp, const FrustumDev &fallback, const uint32_t m, const uint32_t light, const uint32_t face,
                                               const uint32_t cascade, const float *P, const float *V, const uint32_t mask)
{
    float VP[16];
    mat4_mul(P, V, VP);
    fyx_shadow_map &o = mp.maps[m];
    o.light = light;
    o.face = face;
    o.cascade = cascade;
    o.first = 0u;
    o.count = 0u;
    for (int k = 0; k < 16; ++k) o.view_projection[k] = VP[k];
    for (int k = 0; k < 16; ++k) mp.views[(size_t)m * 16 + k] = V[k]; // the observer's view_matrix of the map's instances
    if (frustum_from_view_projection(VP, mp.scratch[m])) {
        to_dev_frustum(mp.scratch[m], mask, FYX_PASS_SHADOW, mp.frusta[m]);
    } else {
        mp.frusta[m] = fallback;
        mp.frusta[m].cam_mask = mask;
    }
}

// the observer of a map's from_graph for the LOD filter (renderer/bundle.rs:873-916): translation, z_near, z_far
__device__ __forceinline__ void map_observer(float *o, const float *t, const float z_near, const float z_far)
{
    o[0] = t[0]; o[1] = t[1]; o[2] = t[2]; o[3] = z_near; o[4] = z_far;
}

// cascade i of a directional light (renderer/shadow/csm.rs:195-249): the light-space box around slice i of the camera
// frustum.  V = the map's look_at_lh, P = its orthographic projection.  obs != nullptr: the cascade's observer
// (shadow/csm.rs:251-265: the look_at_lh eye, the slice's depths after the guard) goes there.
__device__ __forceinline__ void csm_cascade(const CsmCameraDev &cam, const fyx_csm_options &opt, const uint32_t i, const float *light_dir,
                                         const float *light_up, float *V, float *P, float *obs = nullptr)
{
    // csm.rs:181-194: z_values = [z_near, far planes] (Absolute) or [z_near, z_far * fractions] (Relative)
    const float a = i == 0u ? cam.z_near : opt.relative ? FYX_MUL(cam.z_far, opt.splits[i - 1]) : opt.splits[i - 1];
    const float b = opt.relative ? FYX_MUL(cam.z_far, opt.splits[i]) : opt.splits[i];
    const float z_near = a;
    float z_far = b;
    // csm.rs:200-205: MIN_DEPTH_DELTA = 2 * f32::EPSILON
    if (relative_eq(z_far, z_near)) z_far = FYX_ADD(z_far, FYX_MUL(2.3841858e-07f, z_near));
    float M[16];
    camera_projection(cam.projection, cam.m22_or_vertical_size, z_near, z_far, cam.frame_size[0], cam.frame_size[1], P);
    mat4_mul(P, cam.view, M);
    fyx_frustum fr;
    if (!frustum_from_view_projection(M, fr)) fr = cam.fallback;
    float c[3];
    frustum_center(fr, c);
    const float eye[3] = {FYX_ADD(c[0], light_dir[0]), FYX_ADD(c[1], light_dir[1]), FYX_ADD(c[2], light_dir[2])};
    if (obs) map_observer(obs, eye, z_near, z_far);
    look_at_lh(eye, c, light_up, V);
    // AxisAlignedBoundingBox::default + add_point of every light-space corner
    float mn[3] = {3.40282347e+38f, 3.40282347e+38f, 3.40282347e+38f}, mx[3] = {-3.40282347e+38f, -3.40282347e+38f, -3.40282347e+38f};
    for (int k = 0; k < 8; ++k) {
        float t[3];
        transform_point(V, fr.corners[k], t);
        for (int q = 0; q < 3; ++q) {
            if (t[q] < mn[q]) mn[q] = t[q];
            if (t[q] > mx[q]) mx[q] = t[q];
        }
    }
    // csm.rs:235-246: z_mult = 10
    mn[2] = mn[2] < 0.0f ? FYX_MUL(mn[2], 10.0f) : mn[2] / 10.0f;
    mx[2] = mx[2] < 0.0f ? mx[2] / 10.0f : FYX_MUL(mx[2], 10.0f);
    orthographic(mn[0], mx[0], mn[1], mx[1], mn[2], mx[2], P);
}

// What one light of an observer's light list needs for its maps (shadow_light_gate)
struct ShadowLightGate {
    uint32_t cascade;
    float pos[3], upv[3], lookv[3], radius;
};

// The shadow loop's gates for one light record and one observer — its frustum `cam` and translation cam_t
// (renderer/light.rs:509-606): in the observer's light list (renderer/bundle.rs:926-974, as k_cull_lights), cast_shadows,
// the distance gate, is_intersects_sphere, the cascade index; directional lights need csm_enabled.  Returns the light's
// number of maps: 0, 1 (spot), 6 (point: cube faces) or 3 (directional: cascades).
__device__ __forceinline__ uint32_t shadow_light_gate(const NodeArrays &a, const ShadowParams &sp, const ShadowLightDev &L, const FrustumDev &cam,
                                                      const float *cam_t, const bool csm_enabled, const PackedConsts &kc, ShadowLightGate &g)
{
    const uint32_t slot = L.slot, kind = L.kind;
    const uint32_t nf = a.flags[slot];
    constexpr uint32_t need = FYX_NODE_ALIVE | FYX_NODE_LIGHT | FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED;
    const bool dir = kind == FYX_LIGHT_DIRECTIONAL;
    bool ok = (nf & need) == need && (kind == FYX_LIGHT_SPOT || kind == FYX_LIGHT_POINT || (dir && csm_enabled));
    if (ok) {
        const float2 wx = a.wa[0][slot], wy = a.wa[1][slot], wz = a.wa[2][slot];
        ok = frustum_intersects_aabb(cam, wx, wy, wz, kc, aabb_is_tame(wx, wy, wz));
    }
    if (!ok) return 0u;
    const float4 r0 = a.G[0][slot], r1 = a.G[1][slot], r2 = a.G[2][slot];
    float *pos = g.pos;
    pos[0] = r0.w; pos[1] = r1.w; pos[2] = r2.w;          // global_position
    g.upv[0] = r0.y; g.upv[1] = r1.y; g.upv[2] = r2.y;    // up_vector: column 1
    g.lookv[0] = r0.z; g.lookv[1] = r1.z; g.lookv[2] = r2.z; // look_vector: column 2
    // light.rs:510: (light.position - observer.position.translation).norm()
    const float d[3] = {FYX_SUB(pos[0], cam_t[0]), FYX_SUB(pos[1], cam_t[1]), FYX_SUB(pos[2], cam_t[2])};
    const float dist = sqrtf(dot3(d, d));
    const bool spot = kind == FYX_LIGHT_SPOT;
    const float sd = spot ? sp.spot_distance : sp.point_distance;
    // light.rs:529-532, 547-549: cast_shadows && distance_to_camera <= shadows_distance && enabled;
    // light.rs:555-565 (directional): cast_shadows && csm_settings.enabled (checked above), raw radius f32::MAX
    ok = (nf & FYX_NODE_CAST_SHADOWS) && (dir || (dist <= sd && (spot ? sp.spot_enabled : sp.point_enabled)));
    // light.rs:570-572: max(local scale) * raw radius
    float sx = 1.f, sy = 1.f, sz = 1.f;
    if (sp.trs) {
        sx = sp.trs[slot].scale[0];
        sy = sp.trs[slot].scale[1];
        sz = sp.trs[slot].scale[2];
    }
    const float radius = FYX_MUL(fmaxf(fmaxf(sx, sy), sz), dir ? 3.40282347e+38f : L.distance_or_radius);
    g.radius = radius;
    // light.rs:585-587, Frustum::is_intersects_sphere (fyrox-math/src/frustum.rs:336-347)
    bool sphere = true;
    for (int p = 0; p < 6; ++p) {
        const float4 pl = cam.plane[p];
        const float n[3] = {pl.x, pl.y, pl.z};
        const float dd = FYX_ADD(dot3(n, pos), pl.w);
        if (dd < -radius) { sphere = false; break; }
        if (fabsf(dd) < radius) break;
    }
    ok = ok && sphere;
    // light.rs:589-602 (a distance equal to b1 is neither < b1 nor > b1: cascade 2)
    const float b1 = FYX_MUL(sd, 0.2f), b2 = FYX_MUL(sd, 0.4f);
    const float e[3] = {FYX_SUB(cam_t[0], pos[0]), FYX_SUB(cam_t[1], pos[1]), FYX_SUB(cam_t[2], pos[2])};
    const float metric = sqrtf(dot3(e, e));
    g.cascade = (dist < b1 || metric <= radius) ? 0u : (dist > b1 && dist < b2) ? 1u : 2u;
    return ok ? (dir ? 3u : spot ? 1u : 6u) : 0u;
}

// The maps of one light that passed shadow_light_gate, at rows first.. of the map table, each with the render mask `mask`:
// the cascades of `csm` for a directional light, else the spot map or the six cube faces.  obs != nullptr: each map's LOD
// observer goes there as well (mp.pr.obs).
__device__ __forceinline__ void shadow_light_maps(const MapParams &mp, const FrustumDev &fallback, const ShadowLightDev &L, const ShadowLightGate &g,
                                                  const CsmCameraDev &csm, const uint32_t light, const uint32_t first, const uint32_t mask, float *obs)
{
    const float zdir[3] = {0.f, 0.f, 1.f}, ydir[3] = {0.f, 1.f, 0.f};
    const float *pos = g.pos;
    float P[16], V[16];
    if (L.kind == FYX_LIGHT_DIRECTIONAL) {
        // shadow/csm.rs:170-179: light_direction = -up (normalised, else y), light_up = look (normalised, else z)
        float dir[3], up[3];
        try_normalize(g.upv, ydir, dir);
        dir[0] = -dir[0]; dir[1] = -dir[1]; dir[2] = -dir[2];
        try_normalize(g.lookv, zdir, up);
#pragma unroll 1
        for (uint32_t k = 0; k < 3u; ++k) {
            csm_cascade(csm, L.csm, k, dir, up, V, P, obs ? obs + (size_t)(first + k) * 5 : nullptr);
            shadow_map_out(mp, fallback, first + k, light, 0u, k, P, V, mask);
        }
    } else {
        perspective(L.m22, 1.0f, 0.01f, g.radius, P); // z_near 0.01, z_far light_radius (light.rs:702-704, point.rs:167-170)
        if (obs) // light.rs:700-728, shadow/point.rs:162-190: the light's position, z_near 0.01, z_far light_radius
            for (uint32_t k = 0; k < (L.kind == FYX_LIGHT_SPOT ? 1u : 6u); ++k) map_observer(obs + (size_t)(first + k) * 5, pos, 0.01f, g.radius);
        if (L.kind == FYX_LIGHT_SPOT) {
            // light.rs:706-722: look_at_rh(pos, pos - emit_direction, look_vector normalised)
            float emit[3], up[3];
            try_normalize(g.upv, zdir, emit);
            try_normalize(g.lookv, ydir, up);
            const float target[3] = {FYX_SUB(pos[0], emit[0]), FYX_SUB(pos[1], emit[1]), FYX_SUB(pos[2], emit[2])};
            look_at_rh(pos, target, up, V);
            shadow_map_out(mp, fallback, first, light, 0u, g.cascade, P, V, mask);
        } else {
            // shadow/point.rs:172-180: one map per cube face
#pragma unroll 1
            for (uint32_t k = 0; k < 6u; ++k) {
                const float target[3] = {FYX_ADD(pos[0], c_face_look[k][0]), FYX_ADD(pos[1], c_face_look[k][1]), FYX_ADD(pos[2], c_face_look[k][2])};
                const float up[3] = {c_face_up[k][0], c_face_up[k][1], c_face_up[k][2]};
                look_at_rh(pos, target, up, V);
                shadow_map_out(mp, fallback, first + k, light, k, g.cascade, P, V, mask);
            }
        }
    }
}

// PRUNE: each map's LOD observer goes to mp.pr.obs as well
template <bool PRUNE>
__global__ void __launch_bounds__(kBlock) k_shadow_frusta(const NodeArrays a, const MapParams mp, const ShadowParams sp)
{
    __shared__ BlockScan<kBlock> s_scan;
    const uint32_t tid = threadIdx.x;
    pdl_trigger(); // the node pass loads its columns meanwhile
    if (tid == 0) s_scan.base = 0u;
    const PackedConsts kc = packed_consts();
    for (uint32_t base = 0; base < sp.n_lights; base += kBlock) {
        const uint32_t i = base + tid;
        uint32_t n_maps = 0u;
        ShadowLightDev L{};
        ShadowLightGate g;
        if (i < sp.n_lights) {
            L = sp.lights[i];
            n_maps = shadow_light_gate(a, sp, L, sp.cam, sp.cam_t, sp.csm.enabled, kc, g);
        }
        // ordered compaction: maps in light (pool) order
        const uint32_t first = s_scan.place(n_maps);
        if (n_maps) shadow_light_maps(mp, sp.fallback, L, g, sp.csm, a.gidx[L.slot], first, sp.cam.cam_mask, PRUNE ? mp.pr.obs : nullptr);
    }
    if (tid == 0) *mp.n_maps = s_scan.base;
}

// the node's part of from_graph for a map, minus the frustum test: alive, renderable, reachable, globally visible and
// enabled; the shadow forms add cast_shadows, and kFormShadow the render mask against the camera's.  The other forms test
// each map's mask in shadow_in_map.
template <int FORM>
__device__ __forceinline__ bool shadow_candidate(const uint32_t nf, const uint32_t mask, const MapParams &mp)
{
    if (FORM == kFormObservers) return (nf & kNeedBits) == kNeedBits;
    if (FORM == kFormSceneShadow) return (nf & kShadowNeed) == kShadowNeed;
    return (nf & kShadowNeed) == kShadowNeed && (mask & mp.cam_mask) != 0u;
}

// The one predicate of the count and emit passes (and of a static batch's "rendered" in the pruner table): the node is in
// map m's list.  hrow (PRUNE only): the node's row of the pruner table, the maps in which the LOD filter or a static batch
// above it hides it (nullptr = none); hword carries its word of the current 32 maps from one map to the next.  Forms other
// than kFormShadow: the node's render mask against map m's (should_be_rendered, scene/node/mod.rs:231-256).
template <bool PRUNE, int FORM>
__device__ __forceinline__ bool shadow_in_map(const FrustumDev *__restrict__ F, const uint32_t m, const bool cand, const bool test, const bool tame,
                                              const float2 wx, const float2 wy, const float2 wz, const PackedConsts &kc,
                                              const uint32_t *hrow, uint32_t &hword, const uint32_t mask)
{
    bool ok;
    if (FORM != kFormShadow) {
        ok = cand && (mask & F[m].cam_mask) != 0u;
        if (ok && test) ok = frustum_intersects_aabb(F[m], wx, wy, wz, kc, tame);
    } else {
        ok = test ? frustum_intersects_aabb(F[m], wx, wy, wz, kc, tame) : cand;
    }
    if (PRUNE && hrow) {
        if ((m & 31u) == 0u) hword = hrow[m >> 5];
        ok = ok && !((hword >> (m & 31u)) & 1u);
    }
    return ok;
}

// The pruner table of a shadow cull, one launch per hierarchy level's pruners [p_lo, p_hi) (parents first), one thread per
// (pruner, word of 32 maps); drawn in a map = shadow_in_map
template <int FORM>
__global__ void __launch_bounds__(kBlock) k_shadow_pruners(const NodeArrays a, const MapParams mp, const uint32_t p_lo, const uint32_t p_hi)
{
    pdl_wait(); // the map table and its observers
    const uint32_t W = mp.pr.words;
    const uint64_t t = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
    if (t >= (uint64_t)(p_hi - p_lo) * W) return;
    const uint32_t p = p_lo + (uint32_t)(t / W), w = (uint32_t)(t % W);
    const uint32_t slot = mp.pr.slot[p];
    const uint32_t nf = a.flags[slot], mask = a.mask[slot];
    const float2 wx = a.wa[0][slot], wy = a.wa[1][slot], wz = a.wa[2][slot];
    const PackedConsts kc = packed_consts();
    const bool cand = shadow_candidate<FORM>(nf, mask, mp);
    const bool tame = cand && aabb_is_tame(wx, wy, wz);
    const bool test = cand && (nf & FYX_NODE_FRUSTUM_CULLING);
    uint32_t unused = 0u;
    pruner_step(
        a, mp.pr, p, slot, w, *mp.n_maps,
        [&](const uint32_t m) {
            const float *o = mp.pr.obs + (size_t)m * 5;
            return fyx_observer{{o[0], o[1], o[2]}, o[3], o[4]};
        },
        [&](const uint32_t m) { return shadow_in_map<false, FORM>(mp.frusta, m, cand, test, tame, wx, wy, wz, kc, nullptr, unused, mask); });
}

// pass 2: every node read once (flags, mask, box: 32 B; with PRUNE its pruner id: 4 B more) and tested against every map;
// one atomic per (warp, map) with an entry
template <bool PRUNE, int FORM>
__global__ void __launch_bounds__(kBlock) k_shadow_count(const NodeArrays a, const MapParams mp)
{
    const uint32_t slot = blockIdx.x * kBlock + threadIdx.x, lane = threadIdx.x & 31u;
    const bool valid = slot < a.cap;
    uint32_t nf = 0u, mask = 0u, pc = FYX_NONE;
    float2 wx = make_float2(0.f, 0.f), wy = wx, wz = wx;
    if (valid) {
        nf = a.flags[slot];
        mask = a.mask[slot];
        wx = ld_stream(a.wa[0] + slot);
        wy = ld_stream(a.wa[1] + slot);
        wz = ld_stream(a.wa[2] + slot);
        if (PRUNE) pc = mp.pr.col[slot];
    }
    pdl_trigger();
    pdl_wait(); // the map table
    const bool cand = valid && shadow_candidate<FORM>(nf, mask, mp);
    uint32_t any = 0u;
    if (__any_sync(0xFFFFFFFFu, cand)) {
        const PackedConsts kc = packed_consts();
        const bool tame = cand && aabb_is_tame(wx, wy, wz);
        const bool test = cand && (nf & FYX_NODE_FRUSTUM_CULLING);
        const FrustumDev *__restrict__ F = mp.frusta;
        const uint32_t n_maps = *mp.n_maps;
        const uint32_t *hrow = PRUNE && cand ? pruner_row(mp.pr.rows, mp.pr.words, pc) : nullptr;
        uint32_t hword = 0u;
        for (uint32_t m = 0; m < n_maps; ++m) {
            const bool ok = shadow_in_map<PRUNE, FORM>(F, m, cand, test, tame, wx, wy, wz, kc, hrow, hword, mask);
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, ok);
            if (b && lane == 0u) atomicAdd(mp.counts + (size_t)m * kCountStride, (uint32_t)__popc(b));
            any |= b;
        }
    }
    if (lane == 0u) mp.warp_any[slot >> 5] = any;
}

// the lists' places: maps[m].first / count, counts[m] becomes map m's write cursor, total = all entries
__global__ void __launch_bounds__(1024) k_shadow_scan(const MapParams mp)
{
    __shared__ BlockScan<1024u> s_scan;
    const uint32_t tid = threadIdx.x;
    pdl_wait();
    if (tid == 0) s_scan.base = 0u;
    const uint32_t n = *mp.n_maps;
    for (uint32_t base = 0; base < n; base += 1024u) {
        const uint32_t m = base + tid;
        const uint32_t c = m < n ? mp.counts[(size_t)m * kCountStride] : 0u;
        const uint32_t first = s_scan.place(c);
        if (m < n) {
            mp.maps[m].first = first;
            mp.maps[m].count = c;
            mp.counts[(size_t)m * kCountStride] = first;
        }
    }
    if (tid == 0) *mp.total = s_scan.base;
}

// pass 3: the warps that had an entry test again and write their node indices (and, with instances enabled, their slots).
// PRUNE: a warp whose entries would reach past its map's list (first + count) writes nothing and raises E_SHADOW_LIST.
template <bool PRUNE, int FORM>
__global__ void __launch_bounds__(kBlock) k_shadow_emit(const NodeArrays a, const MapParams mp)
{
    const uint32_t slot = blockIdx.x * kBlock + threadIdx.x, lane = threadIdx.x & 31u;
    pdl_wait();
    if (!mp.warp_any[slot >> 5]) return; // warp-uniform
    const bool valid = slot < a.cap;
    uint32_t nf = 0u, mask = 0u, gi = 0u, pc = FYX_NONE;
    float2 wx = make_float2(0.f, 0.f), wy = wx, wz = wx;
    if (valid) {
        nf = a.flags[slot];
        mask = a.mask[slot];
        wx = ld_stream(a.wa[0] + slot);
        wy = ld_stream(a.wa[1] + slot);
        wz = ld_stream(a.wa[2] + slot);
        gi = a.gidx[slot];
        if (PRUNE) pc = mp.pr.col[slot];
    }
    const bool cand = valid && shadow_candidate<FORM>(nf, mask, mp);
    const PackedConsts kc = packed_consts();
    const bool tame = cand && aabb_is_tame(wx, wy, wz);
    const bool test = cand && (nf & FYX_NODE_FRUSTUM_CULLING);
    const FrustumDev *__restrict__ F = mp.frusta;
    const uint32_t n_maps = *mp.n_maps;
    const uint32_t lt = (1u << lane) - 1u;
    const uint32_t *hrow = PRUNE && cand ? pruner_row(mp.pr.rows, mp.pr.words, pc) : nullptr;
    uint32_t hword = 0u;
    for (uint32_t m = 0; m < n_maps; ++m) {
        const bool ok = shadow_in_map<PRUNE, FORM>(F, m, cand, test, tame, wx, wy, wz, kc, hrow, hword, mask);
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, ok);
        if (!b) continue;
        uint32_t at = 0u;
        if (lane == 0u) at = atomicAdd(mp.counts + (size_t)m * kCountStride, (uint32_t)__popc(b));
        at = __shfl_sync(0xFFFFFFFFu, at, 0);
        if (PRUNE && at + (uint32_t)__popc(b) > mp.maps[m].first + mp.maps[m].count) { // warp-uniform
            if (lane == 0u) atomicOr(mp.pr.err, E_SHADOW_LIST);
            continue;
        }
        if (ok) {
            mp.entries[at + __popc(b & lt)] = gi;
            if (mp.entry_slot) mp.entry_slot[at + __popc(b & lt)] = slot;
        }
    }
}

uint32_t launch_shadow_frusta(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ShadowParams &sp, bool pruned)
{
    if (pruned) k_shadow_frusta<true><<<1, kBlock, 0, s>>>(a, mp, sp);
    else k_shadow_frusta<false><<<1, kBlock, 0, s>>>(a, mp, sp);
    return 1u;
}

// The instances of the node passes, by [pruned][form]: the one place that picks one
using NodePass = void (*)(NodeArrays, MapParams);
static const NodePass kCountPass[2][3] = {
    {k_shadow_count<false, kFormShadow>, k_shadow_count<false, kFormObservers>, k_shadow_count<false, kFormSceneShadow>},
    {k_shadow_count<true, kFormShadow>, k_shadow_count<true, kFormObservers>, k_shadow_count<true, kFormSceneShadow>}};
static const NodePass kEmitPass[2][3] = {
    {k_shadow_emit<false, kFormShadow>, k_shadow_emit<false, kFormObservers>, k_shadow_emit<false, kFormSceneShadow>},
    {k_shadow_emit<true, kFormShadow>, k_shadow_emit<true, kFormObservers>, k_shadow_emit<true, kFormSceneShadow>}};
static void (*const kPrunerTable[3])(NodeArrays, MapParams, uint32_t, uint32_t) = {k_shadow_pruners<kFormShadow>, k_shadow_pruners<kFormObservers>,
                                                                                  k_shadow_pruners<kFormSceneShadow>};

uint32_t launch_map_count(cudaStream_t s, const NodeArrays &a, const MapParams &mp, ShadowForm form, const uint32_t *pr_level_off, uint32_t n_levels)
{
    const bool pruned = pr_level_off != nullptr;
    uint32_t n = 0u;
    for (uint32_t l = 0; pruned && l < n_levels; ++l) {
        const uint32_t lo = pr_level_off[l], hi = pr_level_off[l + 1];
        if (hi <= lo) continue;
        launch_pdl(kPrunerTable[form], grid_for((uint64_t)(hi - lo) * mp.pr.words), kBlock, 0, s, a, mp, lo, hi);
        ++n;
    }
    if (a.cap) {
        launch_pdl(kCountPass[pruned][form], grid_for(a.cap), kBlock, 0, s, a, mp);
        ++n;
    }
    return n;
}

uint32_t launch_map_scan(cudaStream_t s, const MapParams &mp)
{
    launch_pdl(k_shadow_scan, 1, 1024, 0, s, mp);
    return 1u;
}

uint32_t launch_map_emit(cudaStream_t s, const NodeArrays &a, const MapParams &mp, ShadowForm form, bool pruned)
{
    if (!a.cap) return 0u;
    launch_pdl(kEmitPass[pruned][form], grid_for(a.cap), kBlock, 0, s, a, mp);
    return 1u;
}

// ------------------------------------------------------------------------------------------------
// N4 shadow maps of the scene's observers (fyx_cull_scene_shadow_casters): the shadow loop of renderer/light.rs:509-782 for
// every observer of the last fyx_cull_scene_observers (render_scene_observer, renderer/mod.rs:964-1120), through the shadow
// maps' node passes in kFormSceneShadow.  A candidate is one (observer, entry of its light list); candidate p is entry p of
// the observers' light lists, which lie one after the other in table order.
// ------------------------------------------------------------------------------------------------
// the observer whose light list holds entry p: the last one whose list starts at or before p (observers with an empty list
// start where the next one does)
__device__ __forceinline__ uint32_t candidate_observer(const SceneShadowParams &ss, const uint32_t p)
{
    uint32_t lo = 0u, hi = ss.n_obs; // table[lo].lights_first <= p < table[hi].lights_first
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (ss.table[mid].lights_first <= p) lo = mid;
        else hi = mid;
    }
    return lo;
}

// the row of the light table (pool order) that holds node's record, FYX_NONE = none
__device__ __forceinline__ uint32_t light_record(const NodeArrays &a, const ShadowParams &sp, const uint32_t node)
{
    uint32_t lo = 0u, hi = sp.n_lights;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const uint32_t n = a.gidx[sp.lights[mid].slot];
        if (n == node) return mid;
        if (n < node) lo = mid + 1u;
        else hi = mid;
    }
    return FYX_NONE;
}

// the hash of a sharing key (light record, cascade, render mask): spot and point maps with equal keys are equal maps
__device__ __forceinline__ uint32_t share_hash(const uint32_t light, const uint32_t cascade, const uint32_t mask)
{
    uint32_t h = light * 0x9E3779B1u ^ (mask * 0x85EBCA77u + cascade * 0xC2B2AE3Du);
    h ^= h >> 15;
    h *= 0x2C1B3C6Du;
    return h ^ (h >> 13);
}

// The camera of observer m's cascades (shadow/csm.rs:179-270 with the observer's projection, view and frame size).  A
// camera's record is found by (kind, node): the records are the probes in pool order, then the cameras in pool order.
__device__ __forceinline__ void observer_csm_camera(const NodeArrays &a, const ShadowParams &sp, const SceneShadowParams &ss, const uint32_t m,
                                                    CsmCameraDev &cam)
{
    const fyx_scene_observer &o = ss.table[m];
    cam.enabled = ss.csm_enabled;
    cam.z_near = o.z_near;
    cam.z_far = o.z_far;
    for (int k = 0; k < 16; ++k) cam.view[k] = o.view[k];
    cam.fallback = sp.csm.fallback;
    if (o.kind == FYX_OBSERVER_CAMERA) {
        const uint64_t want = (1ull << 32) | o.node;
        uint32_t lo = 0u, hi = ss.n_recs;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            const ObserverRecDev &r = ss.recs[mid];
            const uint64_t k = ((uint64_t)(r.kind == FYX_OBSERVER_CAMERA) << 32) | a.gidx[r.slot];
            if (k < want) lo = mid + 1u;
            else hi = mid;
        }
        const ObserverRecDev &R = ss.recs[lo];
        const bool own = R.v[0] != 0.0f || R.v[1] != 0.0f; // a render target's size
        cam.projection = R.mode;
        cam.m22_or_vertical_size = R.m22_or_vertical_size;
        cam.frame_size[0] = own ? R.v[0] : ss.frame_size[0];
        cam.frame_size[1] = own ? R.v[1] : ss.frame_size[1];
    } else {
        // a cube face is square: Projection::matrix uses only w / h (camera.rs:89-106)
        cam.projection = FYX_PROJECTION_PERSPECTIVE;
        cam.m22_or_vertical_size = ss.probe_m22;
        cam.frame_size[0] = cam.frame_size[1] = 1.0f;
    }
}

// One CTA builds the map table and the refs.
//   1. every observer's cascade camera (ss.csm_cams) and every candidate's gate (shadow_light_gate with the observer's
//      frustum and translation);
//   2. a spot or point candidate that gets maps enters its key into the hash (open addressing, linear probing; a slot keeps
//      the smallest candidate of its key);
//   3. in candidate order, one ordered block scan over (new maps, refs): a candidate that is the first
//      of its key, or a directional light, builds its maps; every candidate writes its refs, to its own maps or its key's.
// The work grows with the candidates (observers x lights in their lists; the benchmark scene has 26 x 17 = 442), twice
// 256 at a time: it assumes at most some tens of thousands of candidates, as a one-CTA pass.
__global__ void __launch_bounds__(kBlock) k_scene_shadow_maps(const NodeArrays a, const MapParams mp, const ShadowParams sp, const SceneShadowParams ss)
{
    __shared__ BlockScan<kBlock> s_scan;
    __shared__ uint32_t s_maps, s_refs; // a round scans (new maps << 16 | refs); the two bases are carried apart, in full words
    const uint32_t tid = threadIdx.x;
    pdl_trigger(); // the node pass loads its columns meanwhile
    if (tid == 0) s_maps = s_refs = 0u;
    const PackedConsts kc = packed_consts();
    for (uint32_t m = tid; m < ss.n_obs; m += kBlock) observer_csm_camera(a, sp, ss, m, ss.csm_cams[m]);
    for (uint32_t p = tid; p < ss.n_cand; p += kBlock) {
        SceneShadowCand &C = ss.cand[p];
        const uint32_t m = candidate_observer(ss, p), node = ss.light_entries[p], row = light_record(a, sp, node);
        const fyx_scene_observer &o = ss.table[m];
        C.observer = m;
        C.light = row;
        C.n_maps = C.cascade = 0u;
        C.hslot = FYX_NONE;
        if (row == FYX_NONE) continue; // no record: Unknown (light.rs:560-568)
        ShadowLightGate g;
        C.n_maps = shadow_light_gate(a, sp, sp.lights[row], ss.frusta[m], o.translation, ss.csm_enabled != 0u, kc, g);
        C.cascade = g.cascade;
    }
    __syncthreads();
    for (uint32_t p = tid; p < ss.n_cand; p += kBlock) {
        SceneShadowCand &C = ss.cand[p];
        if (!C.n_maps || sp.lights[C.light].kind == FYX_LIGHT_DIRECTIONAL) continue; // cascades are never shared
        const uint32_t mask = ss.table[C.observer].render_mask;
        for (uint32_t h = share_hash(C.light, C.cascade, mask) & ss.hash_mask;; h = (h + 1u) & ss.hash_mask) {
            const uint32_t q = atomicCAS(ss.hash + h, FYX_NONE, p);
            const SceneShadowCand &Q = ss.cand[q == FYX_NONE ? p : q];
            if (Q.light == C.light && Q.cascade == C.cascade && ss.table[Q.observer].render_mask == mask) {
                if (q != FYX_NONE) atomicMin(ss.hash + h, p);
                C.hslot = h;
                break;
            }
        }
    }
    __syncthreads();
    for (uint32_t base = 0; base < ss.n_cand; base += kBlock) {
        const uint32_t p = base + tid;
        uint32_t n_refs = 0u, n_new = 0u, src = p;
        if (p < ss.n_cand) {
            const SceneShadowCand &C = ss.cand[p];
            n_refs = C.n_maps;
            if (C.hslot != FYX_NONE) src = ss.hash[C.hslot];
            n_new = src == p ? n_refs : 0u;
        }
        // one scan of (new maps << 16 | refs): at most 6 x 256 of either per round
        const uint32_t excl = s_scan.excl(n_new << 16 | n_refs);
        const uint32_t first_map = s_maps + (excl >> 16), first_ref = s_refs + (excl & 0xFFFFu);
        if (n_new) {
            const SceneShadowCand &C = ss.cand[p];
            const ShadowLightDev &L = sp.lights[C.light];
            ShadowLightGate g;
            shadow_light_gate(a, sp, L, ss.frusta[C.observer], ss.table[C.observer].translation, ss.csm_enabled != 0u, kc, g);
            shadow_light_maps(mp, sp.fallback, L, g, ss.csm_cams[C.observer], ss.light_entries[p], first_map, ss.table[C.observer].render_mask, mp.pr.obs);
            ss.cand[p].row = first_map;
        }
        __syncthreads(); // the rows of this round's first candidates
        for (uint32_t k = 0; k < n_refs; ++k) ss.refs[first_ref + k] = fyx_scene_shadow_map{ss.cand[p].observer, ss.cand[src].row + k};
        __syncthreads();
        if (tid == kBlock - 1) {
            s_maps = first_map + n_new;
            s_refs = first_ref + n_refs;
        }
        __syncthreads();
    }
    if (tid == 0) {
        *mp.n_maps = s_maps;
        *ss.n_refs = s_refs;
    }
}

uint32_t launch_scene_shadow_maps(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ShadowParams &sp, const SceneShadowParams &ss)
{
    k_scene_shadow_maps<<<1, kBlock, 0, s>>>(a, mp, sp, ss);
    return 1u;
}

// ------------------------------------------------------------------------------------------------
// N4 scene observers (fyx_cull_scene_observers): ObserversCollection::from_scene (renderer/observer.rs:88-153) with
// Camera::calculate_matrices (scene/camera.rs:454-462), then one from_graph per observer (renderer/mod.rs:1034-1047) through
// the many-map cull's node passes in kFormObservers: the observers are the maps.
// ------------------------------------------------------------------------------------------------
// one observer: its table row, its map row (what k_shadow_scan and the pack read), its frustum with the node's render mask,
// its view matrix and its LOD observer (translation, z_near, z_far)
__device__ __forceinline__ void observer_out(const MapParams &mp, const ObserverParams &op, const uint32_t m, const uint32_t node, const uint32_t kind, const uint32_t face,
                                             const uint32_t mask, const float *t, const float z_near, const float z_far, const float *P,
                                             const float *V)
{
    float VP[16];
    mat4_mul(P, V, VP);
    fyx_scene_observer &o = op.table[m];
    o.node = node;
    o.kind = kind;
    o.face = face;
    o.render_mask = mask;
    o.first = o.count = o.lights_first = o.lights_count = 0u;
    o.environment_map = FYX_NONE;
    for (int k = 0; k < 3; ++k) o.translation[k] = t[k];
    o.z_near = z_near;
    o.z_far = z_far;
    for (int k = 0; k < 16; ++k) {
        o.view[k] = V[k];
        o.projection[k] = P[k];
        o.view_projection[k] = VP[k];
        mp.views[(size_t)m * 16 + k] = V[k];
    }
    fyx_shadow_map &row = mp.maps[m];
    row.light = node;
    row.face = face;
    row.cascade = 0u;
    row.first = row.count = 0u;
    for (int k = 0; k < 16; ++k) row.view_projection[k] = VP[k];
    // renderer/bundle.rs:893-896: from_view_projection_matrix(..).unwrap_or_default()
    if (!frustum_from_view_projection(VP, mp.scratch[m])) mp.scratch[m] = op.fallback;
    to_dev_frustum(mp.scratch[m], mask, 0u, mp.frusta[m]);
    if (mp.pr.obs) map_observer(mp.pr.obs + (size_t)m * 5, t, z_near, z_far);
}

// One CTA: the records in order (due probes' six faces, then cameras), placed by the ordered block scan
__global__ void __launch_bounds__(kBlock) k_observer_views(const NodeArrays a, const MapParams mp, const ObserverParams op)
{
    __shared__ BlockScan<kBlock> s_scan;
    const uint32_t tid = threadIdx.x;
    pdl_trigger();
    if (tid == 0) s_scan.base = 0u;
    for (uint32_t base = 0; base < op.n_recs; base += kBlock) {
        const uint32_t i = base + tid;
        uint32_t n_obs = 0u;
        ObserverRecDev R{};
        if (i < op.n_recs) {
            R = op.recs[i];
            const uint32_t nf = a.flags[R.slot];
            constexpr uint32_t need = FYX_NODE_ALIVE | FYX_NODE_GLOBAL_ENABLED; // observer.rs:91
            if ((nf & need) == need) {
                if (R.kind == FYX_OBSERVER_CAMERA) n_obs = R.enabled ? 1u : 0u;
                else if (R.mode == FYX_PROBE_UPDATE_EACH_FRAME || !R.rendered) n_obs = 6u; // probe.rs:276-290, observer.rs:99-102
            }
            // observer.rs:102 marks the probe updated; here that waits for the call to succeed (k_observer_commit), so a call
            // that fails leaves the probe due
            op.recs[i].emitted = R.kind == FYX_OBSERVER_PROBE_FACE && n_obs ? 1u : 0u;
        }
        const uint32_t first = s_scan.place(n_obs);
        if (n_obs) {
            const uint32_t slot = R.slot, node = a.gidx[slot], mask = a.mask[slot];
            const float4 r0 = a.G[0][slot], r1 = a.G[1][slot], r2 = a.G[2][slot];
            const float pos[3] = {r0.w, r1.w, r2.w};
            float P[16], V[16];
            if (R.kind == FYX_OBSERVER_CAMERA) {
                // camera.rs:454-462: look = column 2, up = column 1, both as they are
                const float target[3] = {FYX_ADD(pos[0], r0.z), FYX_ADD(pos[1], r1.z), FYX_ADD(pos[2], r2.z)};
                const float up[3] = {r0.y, r1.y, r2.y};
                look_at_rh(pos, target, up, V);
                const bool own = R.v[0] != 0.0f || R.v[1] != 0.0f; // a render target's size (camera.rs:813-826)
                camera_projection(R.mode, R.m22_or_vertical_size, R.z_near, R.z_far, own ? R.v[0] : op.frame_size[0],
                                  own ? R.v[1] : op.frame_size[1], P);
                observer_out(mp, op, first, node, FYX_OBSERVER_CAMERA, 0u, mask, pos, R.z_near, R.z_far, P, V);
            } else {
                // observer.rs:104-145: perspective fov 90°, aspect 1 (a cube face); translation = global_rendering_position
                const float t[3] = {FYX_ADD(pos[0], R.v[0]), FYX_ADD(pos[1], R.v[1]), FYX_ADD(pos[2], R.v[2])};
                camera_projection(FYX_PROJECTION_PERSPECTIVE, op.probe_m22, R.z_near, R.z_far, 1.0f, 1.0f, P);
#pragma unroll 1
                for (uint32_t k = 0; k < 6u; ++k) {
                    const float target[3] = {FYX_ADD(t[0], c_face_look[k][0]), FYX_ADD(t[1], c_face_look[k][1]), FYX_ADD(t[2], c_face_look[k][2])};
                    const float up[3] = {c_face_up[k][0], c_face_up[k][1], c_face_up[k][2]};
                    look_at_rh(t, target, up, V);
                    observer_out(mp, op, first + k, node, FYX_OBSERVER_PROBE_FACE, k, mask, t, R.z_near, R.z_far, P, V);
                }
            }
        }
    }
    if (tid == 0) *mp.n_maps = s_scan.base;
}

// The light lists and environment maps of every observer in one pass over the flag column (k_cull_lights and
// k_select_probes for any number of observers): EMIT = false counts each observer's lights and picks its environment map,
// EMIT = true writes the lights at the cursors of k_observer_light_scan.
template <bool EMIT>
__global__ void __launch_bounds__(kBlock) k_observer_lights(const NodeArrays a, const MapParams mp, const ObserverParams op)
{
    const uint32_t slot = blockIdx.x * kBlock + threadIdx.x;
    pdl_wait();
    if (slot >= a.cap) return;
    const uint32_t nf = a.flags[slot];
    constexpr uint32_t need = FYX_NODE_ALIVE | FYX_NODE_LIGHT | FYX_NODE_GLOBAL_VISIBILITY | FYX_NODE_GLOBAL_ENABLED;
    constexpr uint32_t probe = FYX_NODE_ALIVE | FYX_NODE_REFLECTION_PROBE;
    const bool light = (nf & need) == need, env = !EMIT && (nf & probe) == probe;
    if (!light && !env) return;
    const float2 wx = a.wa[0][slot], wy = a.wa[1][slot], wz = a.wa[2][slot];
    const PackedConsts kc = packed_consts();
    const bool tame = aabb_is_tame(wx, wy, wz);
    const uint32_t gi = a.gidx[slot];
    const uint32_t n = *mp.n_maps;
    for (uint32_t m = 0; m < n; ++m) {
        if (light && frustum_intersects_aabb(mp.frusta[m], wx, wy, wz, kc, tame)) {
            uint32_t *c = op.light_counts + (size_t)m * kCountStride;
            if (EMIT) op.light_raw[atomicAdd(c, 1u)] = gi;
            else atomicAdd(c, 1u);
        }
        // renderer/bundle.rs:918-925 (cameras only, renderer/mod.rs:1045-1047): the last probe in pool order containing the observer
        if (env && op.table[m].kind == FYX_OBSERVER_CAMERA) {
            const float px = op.table[m].translation[0], py = op.table[m].translation[1], pz = op.table[m].translation[2];
            if (px >= wx.x && px <= wx.y && py >= wy.x && py <= wy.y && pz >= wz.x && pz <= wz.y) atomicMax(op.best + m, gi + 1u);
        }
    }
}

// One CTA: the table's lists (from the map rows of k_shadow_scan), the light lists' places, the environment maps
__global__ void __launch_bounds__(1024) k_observer_light_scan(const MapParams mp, const ObserverParams op)
{
    __shared__ BlockScan<1024u> s_scan;
    const uint32_t tid = threadIdx.x;
    pdl_wait();
    if (tid == 0) s_scan.base = 0u;
    const uint32_t n = *mp.n_maps;
    for (uint32_t base = 0; base < n; base += 1024u) {
        const uint32_t m = base + tid;
        const uint32_t c = m < n ? op.light_counts[(size_t)m * kCountStride] : 0u;
        const uint32_t first = s_scan.place(c);
        if (m < n) {
            fyx_scene_observer &o = op.table[m];
            o.first = mp.maps[m].first;
            o.count = mp.maps[m].count;
            o.lights_first = first;
            o.lights_count = c;
            o.environment_map = op.best[m] ? op.best[m] - 1u : FYX_NONE;
            op.light_counts[(size_t)m * kCountStride] = first;
        }
    }
    if (tid == 0) *op.light_total = s_scan.base;
}

// One CTA per observer: its light list into ascending node index (pool order, as the reference's pair_iter).  Node
// indices are distinct, so an entry's place is the number of smaller entries.  That is n² compares for a list of n lights,
// n² / 256 per thread: it assumes lists of at most a few thousand lights (4 096 lights = 65 536 compares per thread, tens of µs;
// the observer benchmark's scene has 8 per observer).  A scene whose observers each see far more lights wants a segmented
// radix sort here.
__global__ void __launch_bounds__(kBlock) k_observer_light_sort(const ObserverParams op)
{
    pdl_wait();
    const fyx_scene_observer &o = op.table[blockIdx.x];
    const uint32_t f = o.lights_first, n = o.lights_count;
    const uint32_t *src = op.light_raw + f;
    for (uint32_t i = threadIdx.x; i < n; i += kBlock) {
        const uint32_t v = src[i];
        uint32_t r = 0u;
        for (uint32_t j = 0; j < n; ++j) r += src[j] < v ? 1u : 0u;
        op.light_entries[f + r] = v;
    }
}

__global__ void __launch_bounds__(kBlock) k_observer_commit(ObserverRecDev *recs, const uint32_t n)
{
    const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
    if (i < n && recs[i].emitted) recs[i].rendered = 1u;
}

uint32_t launch_observers_commit(cudaStream_t s, ObserverRecDev *recs, uint32_t n_recs)
{
    if (!n_recs) return 0u;
    k_observer_commit<<<grid_for(n_recs), kBlock, 0, s>>>(recs, n_recs);
    return 1u;
}

uint32_t launch_observer_views(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ObserverParams &op)
{
    k_observer_views<<<1, kBlock, 0, s>>>(a, mp, op);
    return 1u;
}

uint32_t launch_observer_lights(cudaStream_t s, const NodeArrays &a, const MapParams &mp, const ObserverParams &op, bool emit)
{
    if (!a.cap) return 0u;
    if (emit) launch_pdl(k_observer_lights<true>, grid_for(a.cap), kBlock, 0, s, a, mp, op);
    else launch_pdl(k_observer_lights<false>, grid_for(a.cap), kBlock, 0, s, a, mp, op);
    return 1u;
}

uint32_t launch_observer_light_scan(cudaStream_t s, const MapParams &mp, const ObserverParams &op)
{
    launch_pdl(k_observer_light_scan, 1, 1024, 0, s, mp, op);
    return 1u;
}

uint32_t launch_observer_light_sort(cudaStream_t s, const ObserverParams &op, uint32_t n_obs)
{
    if (!n_obs) return 0u;
    launch_pdl(k_observer_light_sort, n_obs, kBlock, 0, s, op);
    return 1u;
}

// the pruners mark their own slots of the column
__global__ void __launch_bounds__(kBlock) k_pruner_mark(const uint32_t n, const uint32_t *pr_slot, uint32_t *col)
{
    const uint32_t p = blockIdx.x * kBlock + threadIdx.x;
    if (p < n) col[pr_slot[p]] = p | kPrSelf;
}

// one hierarchy level: a node that is no pruner takes the nearest pruner on its parent's path; a pruner records it as its
// nearest strict pruner ancestor
__global__ void __launch_bounds__(kBlock) k_pruner_level(const NodeArrays a, const uint32_t lo, const uint32_t hi, uint32_t *col, uint32_t *anc)
{
    const uint32_t slot = lo + blockIdx.x * kBlock + threadIdx.x;
    if (slot >= hi) return;
    const uint32_t p = a.parent[slot];
    const uint32_t pv = p != FYX_NONE ? col[p] : FYX_NONE;
    const uint32_t up = pv != FYX_NONE ? (pv & ~kPrSelf) : FYX_NONE;
    const uint32_t v = col[slot];
    if (v != FYX_NONE) anc[v & ~kPrSelf] = up; // a pruner (the column holds nothing else yet)
    else col[slot] = up;
}

void launch_pruner_mark(cudaStream_t s, uint32_t n_pruners, const uint32_t *pr_slot, uint32_t *col)
{
    if (n_pruners) k_pruner_mark<<<grid_for(n_pruners), kBlock, 0, s>>>(n_pruners, pr_slot, col);
}

void launch_pruner_level(cudaStream_t s, const NodeArrays &a, uint32_t lo, uint32_t hi, uint32_t *col, uint32_t *anc)
{
    if (hi > lo) k_pruner_level<<<grid_for(hi - lo), kBlock, 0, s>>>(a, lo, hi, col, anc);
}

} // namespace fyx
