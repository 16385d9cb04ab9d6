// Dynamic batching's host rules (fyrox_b200/csrc/fyx_dyn_plan.hpp) against the rules stated again here: the device tables in
// push order on random registrations and quad nodes over random forests (with and without a DFS rank, before and after a
// topology change that kills registered and quad nodes, after node surfaces are cut or named skinned); every refusal of the
// checks of fyx_add_dynamic_surface and fyx_set_sprites at its limit, with its code and message; the release of ids and keys;
// the pools' compaction; the placement of a pack's segments at its size limits.  CPU only.  Prints "dyn plan ok" when every
// check held.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <map>
#include <numeric>
#include <random>
#include <string>
#include <vector>

#include "../../fyrox_b200/csrc/fyx_dyn_plan.hpp"
#include "../../fyrox_b200/csrc/fyx_slots.hpp"

using namespace fyx;

static int g_fail = 0;
#define CHECK(cond, ...)                                                                            \
    do {                                                                                            \
        if (!(cond)) {                                                                              \
            if (g_fail++ < 20) {                                                                    \
                fprintf(stderr, "%s:%d: %s: ", __FILE__, __LINE__, #cond);                          \
                fprintf(stderr, __VA_ARGS__);                                                       \
                fprintf(stderr, "\n");                                                              \
            }                                                                                       \
        }                                                                                           \
    } while (0)

// the refusal a check reported
struct Err {
    int32_t code = FYX_OK;
    std::string msg;
};
static auto fail_into(Err &e)
{
    return [&e](int32_t code, const char *fmt, auto... args) {
        char buf[512];
        if constexpr (sizeof...(args) > 0) snprintf(buf, sizeof buf, fmt, args...);
        else snprintf(buf, sizeof buf, "%s", fmt);
        e.code = code;
        e.msg = buf;
        return code;
    };
}

// Mesh::surfaces per node as fyx_set_node_surfaces gives them: count 0 = the default single surface (never skinned)
struct Surfaces {
    std::vector<std::vector<uint8_t>> skinned; // by node: one entry per surface
    std::vector<uint8_t> skinned_node;         // by node: has a skinned fyx surface (fyx_add_skinned_surface)
    DynSurface operator()(uint32_t node, uint32_t ordinal) const
    {
        const std::vector<uint8_t> &s = skinned[node];
        if (ordinal >= std::max<size_t>(s.size(), 1)) return DynSurface::kMissing;
        return !s.empty() && s[ordinal] ? DynSurface::kSkinned : DynSurface::kBatchable;
    }
};

static const fyx_dynamic_layout kLayouts[3] = {{48u, 0u, 12u, 24u}, {12u, 0u, FYX_NONE, FYX_NONE}, {28u, FYX_NONE, 0u, 12u}};
static fyx_dynamic_layout sprite_layout(uint32_t kind) { return fyx_dynamic_layout{kind == FYX_SPRITE_3D ? 40u : 24u, 0u, FYX_NONE, FYX_NONE}; }

// ---- the item plan ------------------------------------------------------------------------------------------------------

// The push order, stated without the planner's code: the dynamic nodes (a quad node, or a node with a registration whose
// surface still exists and is not skinned) by DFS rank, else node index; a node's registered surfaces by ordinal, a quad node
// as one item of ordinal FYX_NONE
static DynItemPlan expected(const DynRegistry &r, const Surfaces &sf, const std::vector<uint32_t> &slot_of_node, uint32_t n_slots,
                            const uint32_t *rank)
{
    std::map<uint32_t, std::map<uint32_t, DynItemDev>> by_node; // node -> ordinal -> item
    for (const DynReg &g : r.regs) {
        const std::vector<uint8_t> &s = sf.skinned[g.node];
        const bool exists = g.ordinal < std::max<size_t>(s.size(), 1), skinned = exists && !s.empty() && s[g.ordinal];
        if (exists && !skinned)
            by_node[g.node][g.ordinal] = DynItemDev{g.node, slot_of_node[g.node], g.batch_key, g.layout, g.n_verts, g.n_tris, g.tri_src, kDynMesh, g.vtx_src};
    }
    for (uint32_t n = 0; n < r.quad_of_node.rec.size(); ++n) {
        const DynQuad &q = r.quad_of_node.rec[n];
        if (q.kind) by_node[n][FYX_NONE] = DynItemDev{n, slot_of_node[n], q.batch_key, q.layout_id, 4u, 2u, 0u, q.kind, 0u};
    }
    std::vector<uint32_t> nodes;
    for (const auto &e : by_node) nodes.push_back(e.first);
    std::stable_sort(nodes.begin(), nodes.end(), [&](uint32_t a, uint32_t b) { return (rank ? rank[a] : a) < (rank ? rank[b] : b); });
    DynItemPlan p;
    p.of_slot.assign(std::max<uint32_t>(n_slots, 1), FYX_NONE);
    uint32_t n_layouts = 0;
    for (uint32_t d = 0; d < nodes.size(); ++d) {
        p.of_slot[slot_of_node[nodes[d]]] = d;
        p.item_first.push_back((uint32_t)p.items.size());
        for (const auto &[ordinal, it] : by_node[nodes[d]]) {
            p.items.push_back(it);
            p.ordinal.push_back(ordinal);
            n_layouts = std::max(n_layouts, it.layout + 1);
            if (it.kind != kDynMesh) ++p.n_quads;
        }
    }
    p.item_first.push_back((uint32_t)p.items.size());
    for (uint32_t l = 0; l < n_layouts; ++l) {
        const fyx_dynamic_layout ly = l < r.layouts.size() ? r.layouts[l] : fyx_dynamic_layout{FYX_NONE, 0, 0, 0};
        p.layouts.push_back(ly.stride == FYX_NONE ? DynLayoutDev{1u, FYX_NONE, FYX_NONE, FYX_NONE}
                                                  : DynLayoutDev{ly.stride, ly.position_offset, ly.normal_offset, ly.tangent_offset});
    }
    return p;
}

static bool same(const DynItemPlan &a, const DynItemPlan &b)
{
    if (a.of_slot != b.of_slot || a.item_first != b.item_first || a.ordinal != b.ordinal || a.n_quads != b.n_quads) return false;
    if (a.items.size() != b.items.size() || a.layouts.size() != b.layouts.size()) return false;
    return memcmp(a.items.data(), b.items.data(), a.items.size() * sizeof(DynItemDev)) == 0 &&
           memcmp(a.layouts.data(), b.layouts.data(), a.layouts.size() * sizeof(DynLayoutDev)) == 0;
}

// a random forest: alive nodes with random earlier parents
static void random_forest(std::mt19937_64 &rng, uint32_t cap, std::vector<uint32_t> &parent, std::vector<uint32_t> &flags)
{
    parent.assign(cap, FYX_NONE);
    flags.assign(cap, FYX_NODE_ALIVE);
    for (uint32_t i = 1; i < cap; ++i)
        if (rng() % 8) parent[i] = (uint32_t)(rng() % i);
    for (uint32_t i = 0; i < cap; ++i)
        if (rng() % 7 == 0) flags[i] = 0;
}

static void test_items(std::mt19937_64 &rng)
{
    int compared = 0, with_quads = 0, with_multi = 0;
    for (int iter = 0; iter < 400; ++iter) {
        const uint32_t cap = 1 + (uint32_t)(rng() % 300);
        std::vector<uint32_t> parent, flags;
        random_forest(rng, cap, parent, flags);
        SlotPlan sp = plan_slots(cap, parent.data(), flags.data());
        Surfaces sf;
        sf.skinned.resize(cap);
        sf.skinned_node.assign(cap, 0);
        for (uint32_t n = 0; n < cap; ++n) {
            if (rng() % 3 == 0) continue; // the default single surface
            sf.skinned[n].resize(rng() % 5);
            for (uint8_t &s : sf.skinned[n]) s = rng() % 6 == 0;
        }
        DynRegistry r;
        Err e;
        const uint32_t tris[3] = {0, 1, 2};
        const int n_regs = (int)(rng() % 400);
        for (int k = 0; k < n_regs; ++k) {
            const uint32_t node = (uint32_t)(rng() % cap), ordinal = (uint32_t)(rng() % 5), key = (uint32_t)(rng() % 12), lid = key % 3;
            const uint32_t nv = 3 + (uint32_t)(rng() % 60), nt = (uint32_t)(rng() % 3);
            DynClaims cl;
            if (r.check_surface(node, ordinal, key, lid, &kLayouts[lid], nv, &nv, nt, tris, sp.slot_of_node, sf, cl, fail_into(e)) == FYX_OK)
                r.add_surface(node, ordinal, key, lid, nv, nt, cl);
        }
        for (int call = 0; call < 3; ++call) {
            std::vector<uint32_t> idx;
            std::vector<fyx_sprite> rec;
            for (uint32_t n = 0; n < cap; ++n)
                if (rng() % 6 == 0) {
                    fyx_sprite s{};
                    s.kind = 1 + (uint32_t)(rng() % 2);
                    s.batch_key = 12 + s.kind;
                    s.layout_id = 2 + s.kind;
                    idx.push_back(n);
                    rec.push_back(s);
                }
            DynClaims cl;
            auto has_surfaces = [&](uint32_t n) { return !sf.skinned[n].empty(); };
            auto skinned = [&](uint32_t n) { return sf.skinned_node[n] != 0; };
            // one call with every listed node that may become a quad node
            std::vector<uint32_t> ok_idx;
            std::vector<fyx_sprite> ok_rec;
            for (size_t k = 0; k < idx.size(); ++k)
                if (sp.slot_of_node[idx[k]] != FYX_NONE && sf.skinned[idx[k]].empty() && !r.registered(idx[k])) {
                    ok_idx.push_back(idx[k]);
                    ok_rec.push_back(rec[k]);
                }
            const int32_t rc = r.check_sprites((uint32_t)ok_idx.size(), ok_idx.data(), ok_rec.data(), sp.slot_of_node, has_surfaces, skinned, cl, fail_into(e));
            CHECK(rc == FYX_OK, "set_sprites refused: %s", e.msg.c_str());
            if (rc == FYX_OK) r.set_sprites((uint32_t)ok_idx.size(), ok_idx.data(), ok_rec.data(), cl);
        }
        for (int phase = 0; phase < 3; ++phase) {
            if (phase == 1) { // a topology change that kills registered and quad nodes and brings others back
                std::vector<uint32_t> flags2 = flags;
                for (uint32_t n = 0; n < cap; ++n)
                    if (rng() % 4 == 0) flags2[n] ^= FYX_NODE_ALIVE;
                SlotPlan sp2 = plan_slots(cap, parent.data(), flags2.data());
                const size_t regs_before = r.regs.size();
                r.topology_changed(sp.slot_of_node, sp2.slot_of_node);
                for (const DynReg &g : r.regs) CHECK(sp2.slot_of_node[g.node] != FYX_NONE, "registration of dead node %u kept", g.node);
                for (uint32_t n = 0; n < r.quad_of_node.rec.size(); ++n)
                    CHECK(!r.quad_of_node.rec[n].kind || (sp.slot_of_node[n] != FYX_NONE && sp2.slot_of_node[n] != FYX_NONE), "quad of node %u kept", n);
                CHECK(r.regs.size() <= regs_before, "registrations grew");
                sp = std::move(sp2);
            }
            if (phase == 2) // node surfaces cut or named skinned
                for (uint32_t n = 0; n < cap; ++n) {
                    if (sf.skinned[n].empty() || rng() % 3) continue;
                    sf.skinned[n].resize(rng() % sf.skinned[n].size());
                    for (uint8_t &s : sf.skinned[n]) s |= rng() % 4 == 0;
                }
            std::vector<uint32_t> rank(cap);
            std::iota(rank.begin(), rank.end(), 0u);
            std::shuffle(rank.begin(), rank.end(), rng);
            for (const uint32_t *rk : {(const uint32_t *)nullptr, (const uint32_t *)rank.data()}) {
                const DynItemPlan got = plan_dyn_items(r, sp.slot_of_node, sp.n_slots(), rk, sf);
                const DynItemPlan want = expected(r, sf, sp.slot_of_node, sp.n_slots(), rk);
                CHECK(same(got, want), "item plan differs (iter %d phase %d rank %d: %zu / %zu items)", iter, phase, rk != nullptr, got.items.size(), want.items.size());
                ++compared;
                with_quads += got.n_quads > 0;
                for (size_t d = 0; d + 1 < got.item_first.size(); ++d) with_multi += got.item_first[d + 1] - got.item_first[d] > 1;
            }
        }
    }
    CHECK(with_quads > 100 && with_multi > 100, "the random sets are too thin (%d plans with quads, %d multi-item nodes)", with_quads, with_multi);
    printf("item plans: %d compared\n", compared);
}

// ---- the checks ---------------------------------------------------------------------------------------------------------

// A registry state without the call stamp: a refused call must leave it as it was
static std::string snapshot(const DynRegistry &r)
{
    std::string s;
    auto put = [&](const void *p, size_t n) { s.append((const char *)p, n); };
    for (const DynReg &g : r.regs) put(&g, sizeof g);
    for (uint64_t p : r.pairs) put(&p, 8);
    for (const DynQuad &q : r.quad_of_node.rec) put(&q, sizeof q);
    for (const fyx_dynamic_layout &l : r.layouts) put(&l, sizeof l);
    for (uint32_t k : r.key_layout) put(&k, 4);
    put(&r.vtx_used, 8);
    put(&r.tri_used, 8);
    put(&r.next_id, 4);
    return s;
}

struct Fixture {
    std::vector<uint32_t> slot_of_node;
    Surfaces sf;
    DynRegistry r;
    // nodes 0..9 alive, node 10 dead; node 3 has two surfaces (ordinal 1 skinned), node 4 a skinned fyx surface, node 5 is a
    // quad node (sprite, key 20, layout id 5), node 6 has a registration (ordinal 0, key 1, layout id 0)
    Fixture()
    {
        slot_of_node = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, FYX_NONE};
        sf.skinned.resize(11);
        sf.skinned[3] = {0, 1};
        sf.skinned_node.assign(11, 0);
        sf.skinned_node[4] = 1;
        fyx_sprite s{};
        s.kind = FYX_SPRITE_3D;
        s.batch_key = 20;
        s.layout_id = 5;
        DynClaims cl;
        Err e;
        const uint32_t node = 5;
        CHECK(sprites(1, &node, &s, cl, e) == FYX_OK, "%s", e.msg.c_str());
        r.set_sprites(1, &node, &s, cl);
        const uint32_t tris[3] = {0, 1, 2};
        DynClaims c2;
        CHECK(surface(6, 0, 1, 0, &kLayouts[0], 3, 1, tris, c2, e) == FYX_OK, "%s", e.msg.c_str());
        r.add_surface(6, 0, 1, 0, 3, 1, c2);
    }
    int32_t surface(uint32_t node, uint32_t ordinal, uint32_t key, uint32_t lid, const fyx_dynamic_layout *ly, uint32_t nv, uint32_t nt,
                    const uint32_t *tris, DynClaims &cl, Err &e)
    {
        static const unsigned char verts[256 * 64] = {};
        return r.check_surface(node, ordinal, key, lid, ly, nv, verts, nt, tris, slot_of_node, sf, cl, fail_into(e));
    }
    int32_t sprites(uint32_t count, const uint32_t *idx, const fyx_sprite *rec, DynClaims &cl, Err &e)
    {
        auto has_surfaces = [&](uint32_t n) { return !sf.skinned[n].empty(); };
        auto skinned = [&](uint32_t n) { return sf.skinned_node[n] != 0; };
        return r.check_sprites(count, idx, rec, slot_of_node, has_surfaces, skinned, cl, fail_into(e));
    }
};

static void expect(int32_t rc, const Err &e, int32_t code, const char *msg, const char *what)
{
    if (code == FYX_OK) CHECK(rc == FYX_OK, "%s: refused (%s)", what, e.msg.c_str());
    else CHECK(rc == code && e.msg == msg, "%s: got %d \"%s\", want %d \"%s\"", what, rc, e.msg.c_str(), code, msg);
}

static void test_surface_checks()
{
    const int32_t BAD = FYX_ERR_INVALID_ARGUMENT;
    const uint32_t tri0[3] = {0, 1, 2};
    struct Case {
        const char *what;
        uint32_t node, ordinal, key, lid;
        fyx_dynamic_layout ly;
        bool null_layout;
        uint32_t nv, nt;
        uint32_t tri_max; // the largest triangle index
        uint64_t tri_used;
        int32_t code;
        const char *msg;
    };
    const fyx_dynamic_layout L0 = kLayouts[0];
    const Case cases[] = {
        {"plain", 7, 0, 2, 1, kLayouts[1], false, 3, 1, 2, 0, FYX_OK, ""},
        {"null layout", 7, 0, 2, 1, kLayouts[1], true, 3, 1, 2, 0, BAD, "layout / verts / triangles is NULL"},
        {"dead node", 10, 0, 2, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "node 10 is not alive"},
        {"node out of range", 11, 0, 2, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "node 11 is not alive"},
        {"255 vertices", 7, 0, 2, 1, kLayouts[1], false, 255, 1, 254, 0, FYX_OK, ""},
        {"256 vertices", 7, 0, 2, 1, kLayouts[1], false, 256, 1, 2, 0, BAD, "256 vertices: only surfaces of fewer than 256 vertices are batched"},
        {"key 2^24 - 1", 7, 0, (1u << 24) - 1, 1, kLayouts[1], false, 3, 1, 2, 0, FYX_OK, ""},
        {"key 2^24", 7, 0, 1u << 24, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "batch key 16777216 too large: keys must be dense (< 2^24)"},
        {"layout id 2^16 - 1", 7, 0, 2, (1u << 16) - 1, kLayouts[1], false, 3, 1, 2, 0, FYX_OK, ""},
        {"layout id 2^16", 7, 0, 2, 1u << 16, kLayouts[1], false, 3, 1, 2, 0, BAD, "layout id 65536 too large: ids must be dense (< 2^16)"},
        {"stride 0", 7, 0, 2, 1, {0u, FYX_NONE, FYX_NONE, FYX_NONE}, false, 3, 1, 2, 0, BAD, "the layout's stride is 0"},
        {"position at the stride's end", 7, 0, 2, 7, {20u, 8u, FYX_NONE, FYX_NONE}, false, 3, 1, 2, 0, FYX_OK, ""},
        {"position past the stride", 7, 0, 2, 7, {20u, 9u, FYX_NONE, FYX_NONE}, false, 3, 1, 2, 0, BAD, "attribute at offset 9 does not fit the stride 20"},
        {"tangent past the stride", 7, 0, 2, 7, {20u, 0u, FYX_NONE, 5u}, false, 3, 1, 2, 0, BAD, "attribute at offset 5 does not fit the stride 20"},
        {"last surface", 3, 0, 2, 1, kLayouts[1], false, 3, 1, 2, 0, FYX_OK, ""},
        {"no such surface", 3, 2, 2, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "node 3 has no surface 2"},
        {"default surface only", 7, 1, 2, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "node 7 has no surface 1"},
        {"skinned surface", 3, 1, 2, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "surface 1 of node 3 is skinned: it is pushed, not batched"},
        {"registered twice", 6, 0, 1, 0, L0, false, 3, 1, 2, 0, BAD, "surface 0 of node 6 is already registered"},
        {"quad node", 5, 0, 2, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "node 5 is a sprite or rectangle (fyx_set_sprites): it has no mesh surfaces"},
        {"same layout id, same layout", 7, 0, 1, 0, L0, false, 3, 1, 2, 0, FYX_OK, ""},
        {"layout id with another layout", 7, 0, 2, 0, kLayouts[1], false, 3, 1, 2, 0, BAD, "layout id 0 was given with another layout"},
        {"quad's layout id with another layout", 7, 0, 2, 5, kLayouts[1], false, 3, 1, 2, 0, BAD, "layout id 5 was given with another layout"},
        {"batch key with another layout id", 7, 0, 1, 1, kLayouts[1], false, 3, 1, 2, 0, BAD,
         "batch key 1 was given with layout 0: one bundle holds one vertex layout"},
        {"quad's batch key", 7, 0, 20, 1, kLayouts[1], false, 3, 1, 2, 0, BAD, "batch key 20 was given with layout 5: one bundle holds one vertex layout"},
        {"last triangle index", 7, 0, 2, 1, kLayouts[1], false, 3, 1, 2, 0, FYX_OK, ""},
        {"triangle index out of range", 7, 0, 2, 1, kLayouts[1], false, 3, 1, 3, 0, BAD, "triangle index 3 out of range (3 vertices)"},
        {"triangles end just below 2^32 words", 7, 0, 2, 1, kLayouts[1], false, 3, 2, 2, (1ull << 32) - 7, FYX_OK, ""},
        {"triangles end at 2^32 words", 7, 0, 2, 1, kLayouts[1], false, 3, 2, 2, (1ull << 32) - 6, BAD,
         "2 triangles do not fit the triangle pool (4294967290 of its 2^32 words in use)"},
        {"no triangles at 2^32 - 1 words", 7, 0, 2, 1, kLayouts[1], false, 3, 0, 2, (1ull << 32) - 1, FYX_OK, ""},
    };
    for (const Case &k : cases) {
        Fixture f;
        f.r.tri_used = std::max(f.r.tri_used, k.tri_used); // no pool behind it: the check reads the use alone
        std::vector<uint32_t> tris(3 * std::max(k.nt, 1u), 0u);
        tris[tris.size() - 1] = k.tri_max;
        const std::string before = snapshot(f.r);
        DynClaims cl;
        Err e;
        const int32_t rc = f.surface(k.node, k.ordinal, k.key, k.lid, k.null_layout ? nullptr : &k.ly, k.nv, k.nt, k.nt ? tris.data() : tri0, cl, e);
        expect(rc, e, k.code, k.msg, k.what);
        CHECK(snapshot(f.r) == before, "%s: the check changed the registry", k.what);
        if (rc == FYX_OK) { // the registration lands at the pools' ends and claims its id and key
            const uint64_t v0 = f.r.vtx_used, t0 = f.r.tri_used;
            const uint32_t id = f.r.add_surface(k.node, k.ordinal, k.key, k.lid, k.nv, k.nt, cl);
            const DynReg &g = f.r.regs.back();
            CHECK(id == 1 && g.vtx_src == v0 && g.tri_src == (uint32_t)t0 && f.r.vtx_used % 16 == 0 && f.r.vtx_used >= v0 + (uint64_t)k.nv * k.ly.stride &&
                      f.r.tri_used == t0 + 3ull * k.nt && f.r.key_layout[k.key] == k.lid && f.r.layouts[k.lid].stride == k.ly.stride,
                  "%s: registration", k.what);
        }
    }
}

static void test_sprite_checks()
{
    const int32_t BAD = FYX_ERR_INVALID_ARGUMENT;
    auto sprite = [](uint32_t kind, uint32_t key, uint32_t lid) {
        fyx_sprite s{};
        s.kind = kind;
        s.batch_key = key;
        s.layout_id = lid;
        return s;
    };
    struct Case {
        const char *what;
        std::vector<uint32_t> idx;
        std::vector<fyx_sprite> rec;
        int32_t code;
        const char *msg;
    };
    const Case cases[] = {
        {"plain", {7, 8}, {sprite(1, 20, 5), sprite(2, 21, 6)}, FYX_OK, ""},
        {"kind 0", {7}, {sprite(0, 20, 5)}, BAD, "record 0: unknown kind 0"},
        {"kind 3", {7, 8}, {sprite(1, 20, 5), sprite(3, 20, 5)}, BAD, "record 1: unknown kind 3"},
        {"dead node", {10}, {sprite(1, 20, 5)}, BAD, "node 10 is not alive"},
        {"node out of range", {11}, {sprite(1, 20, 5)}, BAD, "node 11 is not alive"},
        {"listed twice", {7, 8, 7}, {sprite(1, 20, 5), sprite(1, 20, 5), sprite(1, 20, 5)}, BAD, "node 7 is listed twice"},
        {"key 2^24 - 1", {7}, {sprite(1, (1u << 24) - 1, 5)}, FYX_OK, ""},
        {"key 2^24", {7}, {sprite(1, 1u << 24, 5)}, BAD, "batch key 16777216 too large: keys must be dense (< 2^24)"},
        {"layout id 2^16 - 1", {7}, {sprite(1, 22, (1u << 16) - 1)}, FYX_OK, ""},
        {"layout id 2^16", {7}, {sprite(1, 22, 1u << 16)}, BAD, "layout id 65536 too large: ids must be dense (< 2^16)"},
        {"mesh surfaces", {3}, {sprite(1, 20, 5)}, BAD, "node 3 has mesh surfaces (fyx_set_node_surfaces)"},
        {"skinned", {4}, {sprite(1, 20, 5)}, BAD, "node 4 has a skinned surface"},
        {"registrations", {6}, {sprite(1, 20, 5)}, BAD, "node 6 has dynamic-surface registrations"},
        {"a quad node changes kind", {5}, {sprite(2, 21, 6)}, FYX_OK, ""},
        {"layout id with another layout", {7}, {sprite(2, 21, 5)}, BAD, "layout id 5 was given with another layout"},
        {"mesh layout id", {7}, {sprite(1, 22, 0)}, BAD, "layout id 0 was given with another layout"},
        {"batch key with another layout id", {7}, {sprite(1, 1, 5)}, BAD, "batch key 1 was given with layout 0: one bundle holds one vertex layout"},
        {"key claimed earlier in the call", {7, 8}, {sprite(1, 22, 7), sprite(2, 22, 8)}, BAD,
         "batch key 22 was given with layout 7: one bundle holds one vertex layout"},
        {"layout id claimed earlier in the call", {7, 8}, {sprite(1, 22, 7), sprite(2, 23, 7)}, BAD, "layout id 7 was given with another layout"},
        {"same claim twice in the call", {7, 8}, {sprite(1, 22, 7), sprite(1, 22, 7)}, FYX_OK, ""},
        {"records alone change", {5}, {sprite(1, 20, 5)}, FYX_OK, ""},
    };
    for (const Case &k : cases) {
        Fixture f;
        const std::string before = snapshot(f.r);
        DynClaims cl;
        Err e;
        const int32_t rc = f.sprites((uint32_t)k.idx.size(), k.idx.data(), k.rec.data(), cl, e);
        expect(rc, e, k.code, k.msg, k.what);
        CHECK(snapshot(f.r) == before, "%s: the check changed the registry", k.what);
        if (rc != FYX_OK) continue;
        const bool changed = f.r.set_sprites((uint32_t)k.idx.size(), k.idx.data(), k.rec.data(), cl);
        CHECK(changed == (std::string(k.what) != "records alone change"), "%s: tables changed %d", k.what, changed);
        for (size_t i = 0; i < k.idx.size(); ++i) {
            const DynQuad q = f.r.quad_of_node[k.idx[i]];
            CHECK(q.kind == k.rec[i].kind && q.batch_key == k.rec[i].batch_key && q.layout_id == k.rec[i].layout_id, "%s: record", k.what);
            const fyx_dynamic_layout ly = sprite_layout(q.kind);
            CHECK(f.r.key_layout[q.batch_key] == q.layout_id && !memcmp(&f.r.layouts[q.layout_id], &ly, sizeof ly), "%s: claims", k.what);
        }
    }
    // the duplicate stamp starts again when the call counter wraps
    Fixture f;
    f.r.quad_call = ~0u;
    const uint32_t idx[2] = {7, 8};
    const fyx_sprite rec[2] = {sprite(1, 20, 5), sprite(1, 20, 5)};
    DynClaims cl;
    Err e;
    expect(f.sprites(2, idx, rec, cl, e), e, FYX_OK, "", "call counter wraps");
    expect(f.sprites(2, idx, rec, cl, e), e, FYX_OK, "", "the call after the wrap");
}

// ---- release --------------------------------------------------------------------------------------------------------------

static void test_release()
{
    Fixture f;
    Err e;
    const uint32_t tris[3] = {0, 1, 2};
    DynClaims cl;
    CHECK(f.surface(7, 0, 2, 1, &kLayouts[1], 3, 1, tris, cl, e) == FYX_OK, "%s", e.msg.c_str());
    f.r.add_surface(7, 0, 2, 1, 3, 1, cl);
    // node 7 cleared: key 2 and layout id 1 are free, node 6's stay
    const uint32_t seven = 7;
    f.r.clear_surfaces(1, &seven);
    CHECK(f.r.key_layout[2] == FYX_NONE && f.r.layouts[1].stride == FYX_NONE, "key 2 / layout id 1 not freed");
    CHECK(f.r.key_layout[1] == 0 && f.r.layouts[0].stride == kLayouts[0].stride, "node 6's key / layout id freed");
    CHECK(f.r.registered(6) && !f.r.registered(7) && f.r.pairs.size() == 1, "pairs after the clear");
    // the freed key may come back with another layout id, the freed layout id with another layout
    DynClaims c2;
    expect(f.surface(7, 0, 2, 1, &kLayouts[2], 3, 1, tris, c2, e), e, FYX_OK, "", "freed layout id with another layout");
    DynClaims c3;
    expect(f.surface(7, 0, 2, 3, &kLayouts[2], 3, 1, tris, c3, e), e, FYX_OK, "", "freed key with another layout id");
    // a quad node that changes its key frees the old one; a cleared quad frees its key and layout id
    const uint32_t five = 5;
    fyx_sprite s{};
    s.kind = FYX_SPRITE_RECTANGLE;
    s.batch_key = 30;
    s.layout_id = 9;
    DynClaims c4;
    CHECK(f.sprites(1, &five, &s, c4, e) == FYX_OK, "%s", e.msg.c_str());
    f.r.set_sprites(1, &five, &s, c4);
    CHECK(f.r.key_layout[20] == FYX_NONE && f.r.layouts[5].stride == FYX_NONE && f.r.key_layout[30] == 9, "the quad's old key / layout id");
    f.r.clear_sprites(1, &five);
    CHECK(f.r.key_layout[30] == FYX_NONE && f.r.layouts[9].stride == FYX_NONE && !f.r.quad_of_node[5].kind, "cleared quad");
    // everything cleared
    f.r.clear_surfaces(0, nullptr);
    CHECK(f.r.regs.empty() && f.r.pairs.empty() && f.r.key_layout[1] == FYX_NONE && f.r.layouts[0].stride == FYX_NONE, "clear all");
    // a topology change that kills the registered node frees its key too
    Fixture g;
    std::vector<uint32_t> after = g.slot_of_node;
    after[6] = FYX_NONE;
    after[5] = FYX_NONE;
    g.r.topology_changed(g.slot_of_node, after);
    CHECK(g.r.regs.empty() && g.r.key_layout[1] == FYX_NONE && g.r.key_layout[20] == FYX_NONE && !g.r.quad_of_node[5].kind, "topology");
}

// ---- compaction -----------------------------------------------------------------------------------------------------------

static void test_compaction(std::mt19937_64 &rng)
{
    Fixture f; // node 6: 3 vertices of 48 bytes (144 -> 144), 3 triangle words
    Err e;
    const uint32_t tris[6] = {0, 1, 2, 0, 2, 1};
    CHECK(!plan_dyn_compaction(f.r).compact, "nothing dropped");
    // node 7: 3 vertices of 48 bytes, 1 triangle: dropping it leaves exactly half of both pools
    DynClaims cl;
    CHECK(f.surface(7, 0, 1, 0, &kLayouts[0], 3, 1, tris, cl, e) == FYX_OK, "%s", e.msg.c_str());
    f.r.add_surface(7, 0, 1, 0, 3, 1, cl);
    const uint32_t seven = 7;
    f.r.clear_surfaces(1, &seven);
    CHECK(f.r.vtx_used == 288 && f.r.tri_used == 6, "pool use %llu %llu", (unsigned long long)f.r.vtx_used, (unsigned long long)f.r.tri_used);
    CHECK(!plan_dyn_compaction(f.r).compact, "exactly half dropped");
    f.r.tri_used = 7;
    CHECK(plan_dyn_compaction(f.r).compact, "more than half of the triangle pool dropped");
    f.r.tri_used = 6;
    f.r.vtx_used = 289;
    CHECK(plan_dyn_compaction(f.r).compact, "more than half of the vertex pool dropped");
    // random registrations, random drops: offsets in registration order, each 16-byte aligned and just past the previous one
    for (int iter = 0; iter < 200; ++iter) {
        DynRegistry r;
        std::vector<uint32_t> slot(64);
        std::iota(slot.begin(), slot.end(), 0u);
        Surfaces sf;
        sf.skinned.resize(64);
        std::vector<uint32_t> t(3 * 20, 0u);
        for (int k = 0; k < 100; ++k) {
            const uint32_t node = (uint32_t)(rng() % 64), lid = (uint32_t)(rng() % 3), nv = 1 + (uint32_t)(rng() % 255), nt = (uint32_t)(rng() % 20);
            DynClaims c;
            if (r.check_surface(node, 0, lid, lid, &kLayouts[lid], nv, &nv, nt, t.data(), slot, sf, c, fail_into(e)) == FYX_OK)
                r.add_surface(node, 0, lid, lid, nv, nt, c);
        }
        std::vector<uint32_t> drop;
        for (uint32_t n = 0; n < 64; ++n)
            if (rng() % 4 < (uint64_t)(iter % 4)) drop.push_back(n);
        r.clear_surfaces((uint32_t)drop.size(), drop.data());
        uint64_t live_v = 0, live_t = 0;
        for (const DynReg &g : r.regs) {
            live_v += ((uint64_t)g.n_verts * r.layouts[g.layout].stride + 15) / 16 * 16;
            live_t += 3ull * g.n_tris;
        }
        const DynCompaction p = plan_dyn_compaction(r);
        CHECK(p.compact == (live_v * 2 < r.vtx_used || live_t * 2 < r.tri_used), "compaction rule (iter %d)", iter);
        if (!p.compact) continue;
        CHECK(p.regs.size() == r.regs.size() && p.vtx_used == live_v && p.tri_used == live_t, "fresh pools");
        uint64_t vo = 0, to = 0;
        for (size_t i = 0; i < p.regs.size(); ++i) {
            const DynReg &a = r.regs[i], &b = p.regs[i];
            CHECK(b.id == a.id && b.node == a.node && b.n_verts == a.n_verts && b.vtx_src == vo && b.tri_src == to && b.vtx_src % 16 == 0, "moved registration %zu", i);
            vo += ((uint64_t)a.n_verts * r.layouts[a.layout].stride + 15) / 16 * 16;
            to += 3ull * a.n_tris;
        }
    }
}

// ---- placement ------------------------------------------------------------------------------------------------------------

static void test_placement(std::mt19937_64 &rng)
{
    std::vector<fyx_dynamic_layout> layouts = {kLayouts[0], kLayouts[1], {FYX_NONE, FYX_NONE, FYX_NONE, FYX_NONE}, kLayouts[2]};
    const uint32_t L = (uint32_t)layouts.size();
    // hash capacity per segment: the smallest power of two >= max(64, 2 * items), none for an empty segment
    const uint32_t seg_items[] = {0, 1, 32, 33, 64, 65, 0, 1000, 4096, 4097};
    const uint32_t n_seg = sizeof seg_items / 4;
    std::vector<uint32_t> cnt((size_t)n_seg * L * 3, 0u);
    for (uint32_t g = 0; g < n_seg; ++g) { // items split over layouts 0, 1 and 3; 1 vertex of 12 bytes in layout 1 (pads to 16)
        cnt[((size_t)g * L + 0) * 3] = seg_items[g] / 2;
        cnt[((size_t)g * L + 1) * 3] = seg_items[g] - seg_items[g] / 2;
        cnt[((size_t)g * L + 1) * 3 + 1] = seg_items[g] ? 1 : 0;
        cnt[((size_t)g * L + 0) * 3 + 1] = seg_items[g] / 2 * 7;
        cnt[((size_t)g * L + 0) * 3 + 2] = seg_items[g] / 2 * 5;
        cnt[((size_t)g * L + 1) * 3 + 2] = seg_items[g] ? 3 : 0;
    }
    cnt[((size_t)9 * L + 3) * 3] = 2; // and two items of layout 3 in the last segment
    cnt[((size_t)9 * L + 3) * 3 + 1] = 5;
    DynPlacement p;
    Err e;
    expect(place_dyn_segments(cnt.data(), n_seg, L, layouts, p, fail_into(e)), e, FYX_OK, "", "placement");
    uint64_t items = 0, hash = 0, vb = 0, tr = 0;
    size_t streams = 0;
    for (uint32_t g = 0; g < n_seg; ++g) {
        uint64_t ni = 0;
        CHECK(p.stream0[g] == streams, "stream0[%u]", g);
        for (uint32_t l = 0; l < L; ++l) {
            const uint32_t *k = &cnt[((size_t)g * L + l) * 3];
            CHECK(p.stream_vtx[g * L + l] == vb && p.stream_tri[g * L + l] == tr && vb % 16 == 0, "stream (%u, %u) offsets", g, l);
            if (!k[0]) continue;
            const fyx_dynamic_stream &st = p.streams[streams++];
            CHECK(st.layout_id == l && st.stride == layouts[l].stride && st.n_vertices == k[1] && st.n_triangles == k[2] &&
                      (uintptr_t)st.vertices == vb && (uintptr_t)st.triangles == tr,
                  "stream (%u, %u)", g, l);
            vb = (vb + (uint64_t)k[1] * layouts[l].stride + 15) / 16 * 16;
            tr += k[2];
            ni += k[0];
        }
        uint64_t cap = 1;
        while (cap < std::max<uint64_t>(64, 2 * ni)) cap *= 2;
        CHECK(p.item0[g] == items && p.hash0[g] == hash && p.hmask[g] == cap - 1, "segment %u: item0 %u hash0 %u hmask %u (cap %llu)", g, p.item0[g],
              p.hash0[g], p.hmask[g], (unsigned long long)cap);
        hash += ni ? 2 * cap : 0;
        items += ni;
    }
    CHECK(p.item0[n_seg] == items && p.stream0[n_seg] == streams && streams == p.streams.size() && p.items == items && p.hash == hash &&
              p.vbytes == vb && p.tris == tr,
          "totals");
    CHECK(p.hmask[0] == 63 && p.hmask[1] == 63 && p.hmask[2] == 63 && p.hmask[3] == 127 && p.hmask[4] == 127 && p.hmask[5] == 255 && p.hmask[8] == 8191 &&
              p.hmask[9] == 16383,
          "capacities");
    // no layouts: every segment empty
    expect(place_dyn_segments(nullptr, 3, 0, layouts, p, fail_into(e)), e, FYX_OK, "", "no layouts");
    CHECK(p.item0 == std::vector<uint32_t>(4, 0u) && p.stream0 == std::vector<uint32_t>(4, 0u) && p.streams.empty() && p.hash == 0, "empty placement");

    // the size limits: hash entries < 2^32, items < 2^31, triangle words < 2^32
    struct Lim {
        const char *what;
        std::vector<uint32_t> items, tris; // per segment, all in layout 1
        int32_t code;
        const char *msg;
    };
    const int32_t BAD = FYX_ERR_INVALID_ARGUMENT;
    const Lim lims[] = {
        {"2^29 items in one segment", {1u << 29}, {0}, FYX_OK, ""},
        {"2^29 + 1 items in one segment", {(1u << 29) + 1}, {0}, BAD, "the dynamic batches of one pack are too large (536870913 items)"},
        {"2^30 + 1 items in one segment", {(1u << 30) + 1}, {0}, BAD, "the dynamic batches of one pack are too large (1073741825 items)"},
        {"2^31 items in one segment", {1u << 31}, {0}, BAD, "the dynamic batches of one pack are too large (2147483648 items)"},
        {"2^32 - 1 items in one segment", {~0u}, {0}, BAD, "the dynamic batches of one pack are too large (4294967295 items)"},
        {"hash entries 2^32 - 2^30", {1u << 29, 1u << 28}, {0, 0}, FYX_OK, ""},
        {"hash entries 2^32", {1u << 29, 1u << 29}, {0, 0}, BAD, "the dynamic batches of one pack are too large (1073741824 items)"},
        {"triangle words 2^32 - 1", {1, 1}, {1431655764, 1}, FYX_OK, ""},
        {"triangle words 2^32 + 2", {1, 1}, {1431655765, 1}, BAD, "the dynamic batches of one pack are too large (2 items)"},
    };
    for (const Lim &k : lims) {
        const uint32_t ns = (uint32_t)k.items.size();
        std::vector<uint32_t> c((size_t)ns * L * 3, 0u);
        for (uint32_t g = 0; g < ns; ++g) {
            c[((size_t)g * L + 1) * 3] = k.items[g];
            c[((size_t)g * L + 1) * 3 + 2] = k.tris[g];
        }
        Err e2;
        expect(place_dyn_segments(c.data(), ns, L, layouts, p, fail_into(e2)), e2, k.code, k.msg, k.what);
    }
    // random counts against the same statement
    for (int iter = 0; iter < 300; ++iter) {
        const uint32_t ns = 1 + (uint32_t)(rng() % 12);
        std::vector<uint32_t> c((size_t)ns * L * 3, 0u);
        for (size_t i = 0; i < c.size(); i += 3)
            if (i / 3 % L != 2 && rng() % 3) {
                c[i] = 1 + (uint32_t)(rng() % 300);
                c[i + 1] = c[i] * (uint32_t)(1 + rng() % 200);
                c[i + 2] = c[i] * (uint32_t)(rng() % 100);
            }
        Err e3;
        CHECK(place_dyn_segments(c.data(), ns, L, layouts, p, fail_into(e3)) == FYX_OK, "random placement refused");
        uint64_t it = 0, hs = 0, v = 0;
        for (uint32_t g = 0; g < ns; ++g) {
            uint64_t ni = 0;
            for (uint32_t l = 0; l < L; ++l) {
                CHECK(p.stream_vtx[g * L + l] == v, "random stream offset");
                const uint32_t *k = &c[((size_t)g * L + l) * 3];
                if (k[0]) v = (v + (uint64_t)k[1] * layouts[l].stride + 15) / 16 * 16;
                ni += k[0];
            }
            uint64_t cap = 1;
            while (cap < std::max<uint64_t>(64, 2 * ni)) cap *= 2;
            CHECK(p.item0[g] == it && p.hash0[g] == hs && p.hmask[g] == cap - 1, "random segment");
            hs += ni ? 2 * cap : 0;
            it += ni;
        }
    }
}

int main()
{
    std::mt19937_64 rng(20261018);
    test_items(rng);
    test_surface_checks();
    test_sprite_checks();
    test_release();
    test_compaction(rng);
    test_placement(rng);
    if (g_fail) {
        fprintf(stderr, "%d checks failed\n", g_fail);
        return 1;
    }
    printf("dyn plan ok\n");
    return 0;
}
