"""N3: the camera frusta and the shadow maps share one instance pack (one driver, one scratch, one getter family).

Pins the kernel launches of every pack call, and interleaves packs and getters: camera frusta 0 and 1, the shadow maps, then
frustum 0 again, each getter (host copy, device arrays, surface ordinals, bone blocks) called in mixed order must return bit
for bit what a read taken straight after its own pack returned — whichever segment the host copies held before, and after
another pack reused the scratch."""
import ctypes as C

import numpy as np
import pytest

import fyrox_b200 as fb
from fyrox_b200 import _lib as L
from helpers import camera_frustum
from test_gpu_shadow_casters import ShadowScene, in_view

pytestmark = pytest.mark.gpu

f32 = np.float32
BIG = (200.0, 200.0, 1, 1)
BUNDLE_BYTES = C.sizeof(L.fyx_bundle)


class BoneBlocks(C.Structure):  # fyx_bone_blocks
    _fields_ = [("count", C.c_uint32), ("n_blocks", C.c_uint32), ("block_of_instance", C.c_void_p), ("blocks", C.c_void_p)]


class Getters:
    """The getters of one kind of pack: camera frustum i or shadow map i."""

    def __init__(self, ctx, shadow):
        lib, p = ctx._lib, "fyx_get_shadow_" if shadow else "fyx_get_"
        self.ctx, self.shadow = ctx, shadow
        self.host_fn, self.device_fn = getattr(lib, p + "instances"), getattr(lib, p + "instances_device")
        self.surf_fn = getattr(lib, p + "instance_surfaces")
        self.blocks_fn, self.block_fn = getattr(lib, p + "bone_matrix_blocks_device"), getattr(lib, p + "bone_matrix_block")

    def host(self, i):
        out = L.fyx_instances()
        self.ctx._chk(self.host_fn(self.ctx._h, i, C.byref(out)))
        n, nb = out.count, out.n_bundles
        return (n, nb, C.string_at(out.node, 4 * n), C.string_at(out.sort_index, 8 * n), C.string_at(out.matrices, 128 * n),
                C.string_at(out.bundles, BUNDLE_BYTES * nb))

    def device(self, i):
        out = L.fyx_instances()
        self.ctx._chk(self.device_fn(self.ctx._h, i, C.byref(out)))
        n, nb = out.count, out.n_bundles
        return (n, nb, d2h(out.node, 4 * n), d2h(out.sort_index, 8 * n), d2h(out.matrices, 128 * n), d2h(out.bundles, BUNDLE_BYTES * nb))

    def surfaces(self, i):
        out = L.fyx_instances()
        self.ctx._chk(self.device_fn(self.ctx._h, i, C.byref(out)))
        return self.ctx._instance_surfaces(self.surf_fn, i, out.count).tobytes()

    def blocks(self, i):
        """The device view of the bone blocks, and the host copy of every instance's block."""
        bb = BoneBlocks()
        self.ctx._chk(self.blocks_fn(self.ctx._h, i, C.byref(bb)))
        per = []
        for k in range(bb.count):
            out = np.empty(255 * 16, f32)
            has = C.c_uint32()
            self.ctx._chk(self.block_fn(self.ctx._h, i, k, out.ctypes.data_as(C.c_void_p), C.byref(has)))
            per.append(out.tobytes() if has.value else None)
        return bb.count, bb.n_blocks, d2h(bb.block_of_instance, 4 * bb.count), d2h(bb.blocks, 255 * 64 * bb.n_blocks), per

    def all(self, i):
        return {"host": self.host(i), "device": self.device(i), "surfaces": self.surfaces(i), "blocks": self.blocks(i)}


def d2h(ptr, nbytes):
    """Bytes of device memory (the library's arrays are complete: every pack ends with a synchronisation)."""
    import torch

    if not nbytes:
        return b""

    class Dev:
        __cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}

    return torch.as_tensor(Dev(), device="cuda").cpu().numpy().tobytes()


@pytest.fixture()
def scene(ctx):
    """3000 nodes in 41 bundles, 16 spot and point lights in view of the camera, 40 meshes with one to three surfaces (some
    skinned), instances enabled; returns the two camera frusta."""
    rng = np.random.default_rng(951)
    sc = ShadowScene(rng, 3000, 16, spread=12.0, depth_z=(-30.0, -2.0), kinds=(1, 2), p_cast=1.0)
    in_view(rng, sc)
    sc.load(ctx)
    ctx.set_bundle_ids(rng.integers(0, 41, sc.n).astype(np.uint32))
    renderable = np.flatnonzero((sc.flags & fb.NODE_RENDERABLE) != 0)
    meshes = rng.choice(renderable[renderable > 0], 40, replace=False).tolist()
    surfaces = []
    for i, mesh in enumerate(meshes):
        lst = []
        for s in range(int(rng.integers(1, 4))):
            sid = None
            if i % 3 != 2 and s != 1:
                bones = rng.choice(np.arange(1, sc.n), int(rng.integers(1, 6)), replace=False).astype(np.uint32)
                sid = ctx.add_skinned_surface(mesh, bones, np.tile(np.eye(4, dtype=f32).reshape(16), (bones.size, 1)), None, n_verts=0)
            lst.append((int(rng.integers(41, 50)), sid))
        surfaces.append(lst)
    ctx.set_node_surfaces(meshes, surfaces)
    ctx.update_transforms(fb.UPDATE_ALL)
    ctx.build_palettes()
    ctx.enable_instances()
    return [camera_frustum(zfar=150.0), camera_frustum(target=(0.2, 0.1, -1.0), fovy=np.deg2rad(40.0), zfar=60.0)]


def launches(ctx, fn):
    n = ctx.kernel_launch_count()
    fn()
    return ctx.kernel_launch_count() - n


def test_kernel_launches_of_every_pack(ctx, scene):
    (fo, ff), _ = scene
    ctx.cull([ff])
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *BIG)
    view, vp = np.eye(4, dtype=f32).reshape(16), np.eye(4, dtype=f32).reshape(16)
    ctx.pack_instances(0, view, vp)  # the first pack uploads the per-slot tables
    assert launches(ctx, lambda: ctx.pack_instances(0, view, vp)) == 3  # keys, one-CTA scan, scatter
    assert launches(ctx, lambda: ctx.pack_bone_matrices(0)) == 2  # block index, blocks
    ctx.pack_shadow_instances()
    n_maps = len(ctx.get_shadow_maps()[0])
    assert n_maps > 0 and ctx.get_shadow_maps()[1].size > 0
    assert launches(ctx, ctx.pack_shadow_instances) == 5  # one group: keys, three scan kernels, scatter
    assert launches(ctx, ctx.pack_shadow_bone_matrices) == 1  # one CTA per surface
    assert sum(ctx.get_shadow_instances(k)["node"].size for k in range(n_maps)) > 0
    ctx.cull([ff], cam_mask=[0])  # no node is seen
    assert ctx.get_visible(0).size == 0
    assert launches(ctx, lambda: ctx.pack_instances(0, view, vp)) == 1  # the scan alone
    assert ctx.pack_instances(0, view, vp)["node"].size == 0


def test_packs_and_getters_interleaved(ctx, scene):
    (fo0, ff0), (fo1, ff1) = scene
    cam, sh = Getters(ctx, False), Getters(ctx, True)
    views = [(np.eye(4, dtype=f32).reshape(16), np.eye(4, dtype=f32).reshape(16)) for _ in range(2)]
    views[1][0][12:15] = (0.5, -0.25, 2.0)  # a translated observer: other sort indices
    ctx.cull([ff0, ff1])
    ctx.cull_shadow_casters(0, np.zeros(3, f32), *BIG)

    def pack_camera(f):
        ctx._chk(ctx._lib.fyx_pack_instances(ctx._h, f, views[f][0].ctypes.data, views[f][1].ctypes.data))
        ctx.pack_bone_matrices(f)
        return cam.all(f)

    want = {("cam", 0): pack_camera(0), ("cam", 1): pack_camera(1)}
    ctx.pack_shadow_instances()
    ctx.pack_shadow_bone_matrices()
    n_maps = len(ctx.get_shadow_maps()[0])
    assert n_maps >= 4
    for k in range(n_maps):
        want[("sh", k)] = sh.all(k)
    assert want[("cam", 0)]["host"][0] > 0 and want[("cam", 1)]["host"][0] > 0
    assert sum(want[("sh", k)]["host"][0] for k in range(n_maps)) > 0
    assert any(b is not None for k in range(n_maps) for b in want[("sh", k)]["blocks"][4])
    assert any(b is not None for b in want[("cam", 0)]["blocks"][4])
    # frustum 0 again: the scratch is reused; the order inside a bundle may change, so its new reading is the reference
    want[("cam", 0)] = pack_camera(0)
    j, k = 1, n_maps - 2
    order = [("sh", k, "host"), ("cam", 1, "device"), ("sh", j, "host"), ("sh", k, "host"), ("cam", 0, "host"), ("sh", j, "surfaces"),
             ("cam", 1, "host"), ("sh", k, "device"), ("cam", 0, "surfaces"), ("sh", k, "surfaces"), ("sh", j, "blocks"),
             ("cam", 0, "device"), ("cam", 1, "surfaces"), ("sh", j, "host"), ("cam", 0, "blocks"), ("sh", 0, "host"), ("sh", k, "host"),
             ("cam", 1, "blocks"), ("sh", j, "device"), ("cam", 0, "host"), ("sh", n_maps - 1, "surfaces"), ("sh", k, "surfaces")]
    for kind, i, getter in order:
        g = sh if kind == "sh" else cam
        assert getattr(g, getter)(i) == want[(kind, i)][getter], (kind, i, getter)
    for k in range(n_maps):  # every map once more, after all of that
        assert sh.all(k) == want[("sh", k)], k
