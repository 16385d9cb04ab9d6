// The skinning-table planner of fyx_commit_surfaces (fyrox_b200/csrc/fyx_skin_plan.hpp) against the rules stated again here:
// on random surface lists over random forests (dead and out-of-range mesh nodes and bones, several surfaces per mesh node,
// vertex counts around the tile sizes, with no DFS rank, a valid one, a reversed one and one of the wrong length) and on the
// skinned units of scenegen's scenes.  CPU only.  Prints "skin plan ok" when every check held.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <map>
#include <random>
#include <vector>

#include "../../fyrox_b200/csrc/fyx_skin_plan.hpp"
#include "../../fyrox_b200/csrc/fyx_slots.hpp"
#include "../../fyrox_b200/csrc/scenegen.h"

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

static bool same_tile(const SkinTile &a, const SkinTile &b)
{
    return a.bone_off == b.bone_off && a.n_bones == b.n_bones && a.quad_start == b.quad_start && a.n_quads == b.n_quads &&
           a.n_shapes == b.n_shapes && a.bs_off == b.bs_off && a.bs_blocks == b.bs_blocks && a.w_off == b.w_off &&
           a.local_quad0 == b.local_quad0 && a.vcoded[0] == b.vcoded[0] && a.vcoded[1] == b.vcoded[1] && a.vcoded[2] == b.vcoded[2];
}

struct Scene {
    std::vector<uint32_t> parent, flags;
    std::vector<SkinSurface> surfaces;
};

// A surface appended the way fyx_add_skinned_surface places it: palette entries and vertices (padded to 4) after the last
static void append(Scene &s, uint32_t mesh, std::vector<uint32_t> bones, uint32_t n_verts, uint32_t n_shapes, std::mt19937_64 &rng)
{
    SkinSurface sf;
    sf.mesh_node = mesh;
    sf.bones = std::move(bones);
    sf.bone_off = s.surfaces.empty() ? 0 : s.surfaces.back().bone_off + s.surfaces.back().n_bones();
    sf.n_verts = n_verts;
    sf.vert_off = s.surfaces.empty() ? 0 : s.surfaces.back().vert_off + ((s.surfaces.back().n_verts + 3ull) & ~3ull);
    if (n_shapes && n_verts) {
        sf.n_shapes = n_shapes;
        sf.bs_blocks = (n_verts + 127) / 128;
        sf.bs_off = rng() % 100000;
        sf.w_off = (uint32_t)(rng() % 5000);
    }
    s.surfaces.push_back(std::move(sf));
}

// The rules, stated without the planner's code
static SkinPlan expected(const std::vector<SkinSurface> &surfaces, const std::vector<uint32_t> &slot_of_node, uint32_t n_slots,
                         const uint32_t *rank)
{
    const uint64_t n_nodes = slot_of_node.size();
    auto slot = [&](uint32_t node) { return node < n_nodes ? slot_of_node[node] : FYX_NONE; };
    SkinPlan p;
    for (const SkinSurface &sf : surfaces)
        for (uint32_t b : sf.bones) p.bone_slot.push_back(slot(b));
    // tiles: quads = ceil(n_verts / 4) split into ceil(quads / kTileQuads) tiles of ceil(quads / tiles) quads, the last one shorter
    for (const SkinSurface &sf : surfaces) {
        const uint32_t quads = (sf.n_verts + 3) / 4;
        if (!quads) continue;
        const uint32_t nt = (quads + kTileQuads - 1) / kTileQuads, per = (quads + nt - 1) / nt;
        for (uint32_t q0 = 0; q0 < quads; q0 += per)
            p.tiles.push_back(SkinTile{sf.bone_off, sf.n_bones(), (uint32_t)(sf.vert_off / 4) + q0, std::min(per, quads - q0), sf.n_shapes,
                                       (uint32_t)sf.bs_off, sf.bs_blocks, sf.w_off, q0, {0, 0, 0}});
    }
    // the fold: a surface with bones on an alive mesh node adds its bones, in list order, to its node's entry; the entries are
    // in the order their nodes first appear
    std::vector<uint32_t> order;
    std::map<uint32_t, std::vector<uint32_t>> bones_of;
    for (const SkinSurface &sf : surfaces) {
        if (sf.bones.empty() || slot(sf.mesh_node) == FYX_NONE) continue;
        if (!bones_of.count(sf.mesh_node)) order.push_back(sf.mesh_node);
        std::vector<uint32_t> &v = bones_of[sf.mesh_node];
        v.insert(v.end(), sf.bones.begin(), sf.bones.end());
    }
    p.fold_begin.push_back(0);
    for (uint32_t m : order) {
        p.fold_node.push_back(slot(m));
        for (uint32_t b : bones_of[m]) {
            p.fold_bone.push_back(slot(b));
            const bool late = rank && slot(b) != FYX_NONE && rank[b] > rank[m];
            p.stale_idx.push_back(late ? (uint32_t)p.late_slot.size() : FYX_NONE);
            if (late) p.late_slot.push_back(slot(b));
        }
        p.fold_begin.push_back((uint32_t)p.fold_bone.size());
    }
    p.surf_of_slot.assign(std::max(n_slots, 1u), FYX_NONE);
    for (size_t s = surfaces.size(); s-- > 0;)
        if (!surfaces[s].bones.empty() && slot(surfaces[s].mesh_node) != FYX_NONE) p.surf_of_slot[slot(surfaces[s].mesh_node)] = (uint32_t)s;
    p.surf_bones.assign(std::max<size_t>(surfaces.size(), 1), SurfBones{0, 0});
    for (size_t s = 0; s < surfaces.size(); ++s) p.surf_bones[s] = SurfBones{surfaces[s].bone_off, surfaces[s].n_bones()};
    for (const SkinSurface &sf : surfaces) {
        if (sf.n_verts) p.max_bones = std::max(p.max_bones, sf.n_bones());
        if (sf.n_verts && sf.n_shapes) p.any_blend_shapes = true;
    }
    return p;
}

// rank == nullptr: no rank given
static void check(const Scene &sc, const std::vector<uint32_t> *rank, const char *what)
{
    const SlotPlan sp = plan_slots((uint32_t)sc.parent.size(), sc.parent.data(), sc.flags.data());
    const uint32_t *r = rank ? valid_dfs_rank(*rank, sp.slot_of_node.size()) : nullptr;
    const SkinPlan got = plan_skin(sc.surfaces, sp.slot_of_node, sp.n_slots(), r);
    const SkinPlan want = expected(sc.surfaces, sp.slot_of_node, sp.n_slots(), r);
    CHECK(got.bone_slot == want.bone_slot, "%s: bone_slot differs", what);
    CHECK(got.fold_node == want.fold_node, "%s: fold_node differs (%zu vs %zu meshes)", what, got.fold_node.size(), want.fold_node.size());
    CHECK(got.fold_begin == want.fold_begin, "%s: fold_begin differs", what);
    CHECK(got.fold_bone == want.fold_bone, "%s: fold_bone differs", what);
    CHECK(got.stale_idx == want.stale_idx, "%s: stale_idx differs", what);
    CHECK(got.late_slot == want.late_slot, "%s: late_slot differs (%zu vs %zu late bones)", what, got.late_slot.size(), want.late_slot.size());
    CHECK(got.surf_of_slot == want.surf_of_slot, "%s: surf_of_slot differs", what);
    CHECK(got.surf_bones.size() == want.surf_bones.size(), "%s: %zu palette ranges, want %zu", what, got.surf_bones.size(), want.surf_bones.size());
    for (size_t s = 0; s < std::min(got.surf_bones.size(), want.surf_bones.size()); ++s)
        CHECK(got.surf_bones[s].bone_off == want.surf_bones[s].bone_off && got.surf_bones[s].n_bones == want.surf_bones[s].n_bones,
              "%s: palette range of surface %zu", what, s);
    CHECK(got.max_bones == want.max_bones, "%s: max_bones %u, want %u", what, got.max_bones, want.max_bones);
    CHECK(got.any_blend_shapes == want.any_blend_shapes, "%s: any_blend_shapes", what);
    CHECK(got.tiles.size() == want.tiles.size(), "%s: %zu tiles, want %zu", what, got.tiles.size(), want.tiles.size());
    for (size_t t = 0; t < std::min(got.tiles.size(), want.tiles.size()); ++t)
        CHECK(same_tile(got.tiles[t], want.tiles[t]), "%s: tile %zu (quad %u + %u, want %u + %u)", what, t, got.tiles[t].quad_start,
              got.tiles[t].n_quads, want.tiles[t].quad_start, want.tiles[t].n_quads);
    // every surface's tiles cover its quads exactly once, in order, each of at most kTileQuads quads
    size_t at = 0;
    for (size_t s = 0; s < sc.surfaces.size(); ++s) {
        const SkinSurface &sf = sc.surfaces[s];
        const uint64_t q0 = sf.vert_off / 4, end = q0 + (sf.n_verts + 3) / 4;
        uint64_t q = q0;
        while (q < end && at < got.tiles.size()) {
            const SkinTile &t = got.tiles[at++];
            CHECK(t.quad_start == q && t.local_quad0 == q - q0 && t.n_quads >= 1 && t.n_quads <= kTileQuads && t.bone_off == sf.bone_off,
                  "%s: surface %zu: tile at quad %u + %u, want one at %llu", what, s, t.quad_start, t.n_quads, (unsigned long long)q);
            q += t.n_quads;
        }
        CHECK(q == end, "%s: surface %zu: tiles end at quad %llu, not %llu", what, s, (unsigned long long)q, (unsigned long long)end);
    }
    CHECK(at == got.tiles.size(), "%s: %zu tiles past the last surface", what, got.tiles.size() - at);
}

// pre-order rank of a forest, children in node-index order; dead nodes are ranked after the alive ones
static std::vector<uint32_t> dfs_rank(const Scene &sc)
{
    const uint32_t n = (uint32_t)sc.parent.size();
    auto alive = [&](uint32_t i) { return i < n && (sc.flags[i] & FYX_NODE_ALIVE); };
    std::vector<std::vector<uint32_t>> kids(n);
    std::vector<uint32_t> roots, rank(n, FYX_NONE), stack;
    for (uint32_t i = 0; i < n; ++i)
        if (alive(i)) (alive(sc.parent[i]) ? kids[sc.parent[i]] : roots).push_back(i);
    uint32_t next = 0;
    for (uint32_t r : roots) {
        stack.assign(1, r);
        while (!stack.empty()) {
            const uint32_t x = stack.back();
            stack.pop_back();
            rank[x] = next++;
            for (size_t k = kids[x].size(); k-- > 0;) stack.push_back(kids[x][k]);
        }
    }
    for (uint32_t &r : rank)
        if (r == FYX_NONE) r = next++;
    return rank;
}

static void check_ranks(const Scene &sc, const char *what)
{
    char w[160];
    check(sc, nullptr, what);
    std::vector<uint32_t> r = dfs_rank(sc);
    snprintf(w, sizeof w, "%s, DFS rank", what);
    check(sc, &r, w);
    for (uint32_t &x : r) x = (uint32_t)r.size() - 1 - x;
    snprintf(w, sizeof w, "%s, reversed rank", what);
    check(sc, &r, w);
    r.push_back(0);
    snprintf(w, sizeof w, "%s, rank of the wrong length", what);
    check(sc, &r, w);
}

// a random forest (parents earlier or out of range, some nodes dead) with random surfaces on it
static Scene random_scene(std::mt19937_64 &rng, uint32_t n, uint32_t n_surfaces)
{
    Scene sc;
    sc.parent.resize(n);
    sc.flags.assign(n, FYX_NODE_ALIVE);
    for (uint32_t i = 0; i < n; ++i) {
        sc.parent[i] = (i == 0 || rng() % 10 == 0) ? FYX_NONE : (uint32_t)(rng() % i);
        if (rng() % 8 == 0) sc.flags[i] = 0;
        if (rng() % 40 == 0) sc.parent[i] = n + (uint32_t)(rng() % 3);
    }
    static const uint32_t kVerts[] = {4, 8192, 2 * 8192, 3 * 8192, 8 * 8192}; // each also one to three either side
    std::vector<uint32_t> meshes; // a few mesh nodes carry several surfaces
    for (uint32_t s = 0; s < n_surfaces; ++s) {
        uint32_t mesh;
        const uint32_t pick = (uint32_t)(rng() % 10);
        if (pick == 0) mesh = n + (uint32_t)(rng() % 4); // out of range
        else if (pick < 4 && !meshes.empty()) mesh = meshes[rng() % meshes.size()];
        else mesh = (uint32_t)(rng() % n);
        meshes.push_back(mesh);
        const uint32_t nb = rng() % 6 == 0 ? 0u : 1u + (uint32_t)(rng() % (rng() % 2 ? 8 : 255));
        std::vector<uint32_t> bones(nb);
        for (uint32_t &b : bones) {
            const uint32_t k = (uint32_t)(rng() % 20);
            b = k == 0 ? FYX_NONE : (k == 1 ? n + (uint32_t)(rng() % 5) : (k == 2 ? mesh : (uint32_t)(rng() % n)));
        }
        uint32_t nv = 0;
        if (nb && rng() % 6) {
            const uint32_t k = (uint32_t)(rng() % 4);
            if (k == 0) nv = 1 + (uint32_t)(rng() % 9000);
            else nv = kVerts[rng() % 5] + (uint32_t)(rng() % 7) - 3;
        }
        append(sc, mesh, std::move(bones), nv, rng() % 4 == 0 ? 1 + (uint32_t)(rng() % 8) : 0, rng);
    }
    return sc;
}

// the topology and the skinned units of a scenegen scene (a whole one: rank 0 of 1), each unit's bones in scenegen's order
static Scene scenegen_scene(uint32_t n_nodes, uint32_t n_units, uint32_t bones, uint32_t verts)
{
    sg_config cfg{0xF1A0C5, n_nodes, n_units, bones, verts, 0, 1};
    sg_scene *s = sg_create(&cfg);
    Scene sc;
    CHECK(s, "scenegen refused %u nodes, %u units of %u bones", n_nodes, n_units, bones);
    if (!s) return sc;
    const uint32_t cap = sg_capacity(s);
    sc.parent.assign(sg_parent(s), sg_parent(s) + cap);
    sc.flags.assign(sg_flags(s), sg_flags(s) + cap);
    std::mt19937_64 rng(1);
    for (uint32_t u = 0; u < sg_n_units(s); ++u)
        append(sc, sg_unit_mesh_node(s, u), std::vector<uint32_t>(sg_unit_bone_nodes(s, u), sg_unit_bone_nodes(s, u) + bones), verts, 0, rng);
    sg_free(s);
    return sc;
}

int main()
{
    std::mt19937_64 rng(20261018);
    char what[128];
    check_ranks(Scene{}, "no nodes, no surfaces");
    {
        Scene sc{{FYX_NONE, 0, 0}, {FYX_NODE_ALIVE, FYX_NODE_ALIVE, 0}, {}};
        append(sc, 1, {}, 0, 0, rng);                    // no bones, no vertices
        append(sc, 2, {0, 1}, 8, 0, rng);                // dead mesh node: no fold entry, no surf_of_slot
        append(sc, 1, {0, 2, FYX_NONE, 7, 1}, 9, 2, rng); // dead, NONE, out-of-range and self bones keep their fold entries
        append(sc, 5, {0}, 3, 0, rng);                   // mesh node out of range
        check_ranks(sc, "hand-made");
    }
    for (int t = 0; t < 400; ++t) {
        const uint32_t n = 1 + (uint32_t)(rng() % (t < 300 ? 60 : 5000));
        const Scene sc = random_scene(rng, n, (uint32_t)(rng() % (t < 300 ? 12 : 200)));
        snprintf(what, sizeof what, "random scene %d (%u nodes, %zu surfaces)", t, n, sc.surfaces.size());
        check_ranks(sc, what);
    }
    // scenegen's units: the C3 workload (1 M nodes, 10 k units) and C4's proportions (200 nodes per unit) at 1 M nodes
    const uint32_t sg[][4] = {{1000000, 10000, 64, 5000}, {1000000, 5000, 64, 5000}, {100000, 200, 255, 8193}, {30000, 300, 1, 3}};
    for (auto &c : sg) {
        snprintf(what, sizeof what, "scenegen %u nodes, %u units of %u bones, %u vertices", c[0], c[1], c[2], c[3]);
        check_ranks(scenegen_scene(c[0], c[1], c[2], c[3]), what);
    }
    if (g_fail) {
        fprintf(stderr, "%d checks failed\n", g_fail);
        return 1;
    }
    printf("skin plan ok\n");
    return 0;
}
