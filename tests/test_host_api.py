"""CPU-side tests of the product's host logic and C-ABI surface (no kernel is launched here)."""
import ctypes as C
import json
import os
import numpy as np
import pytest

import util
from util import orc, gltf_ref
import vpt_b200 as pt


def test_library_loads_and_exports_every_declared_symbol():
    L = pt.lib()
    names = pt.declared_symbols()
    assert len(names) >= 45
    for n in names:
        assert hasattr(L, n), f"include/b200pt.h declares {n} but libb200pt.so does not export it"
    assert b"sm_90a" in L.b200pt_version()


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    h = C.c_void_p()
    r = pt.lib().b200pt_create(0, C.byref(h))
    assert r == pt.ERR_NO_DEVICE and not h.value          # fails loudly: there is no CPU rendering path
    with pytest.raises(pt.B200ptError):
        pt.PathTracer(0)


def test_null_arguments_are_rejected_not_crashed():
    L = pt.lib()
    assert L.b200pt_create(0, None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_destroy(None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_path_trace(None, 1, 0, None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_set_scene_file(None, b"x") == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_add_volume(None, None) == pt.ERR_WRONG_ARGUMENTS      # homogeneous volumes are implemented: a null volume is a bad argument
    assert L.b200pt_add_density_data_to_volume(None, 0, None) == pt.ERR_NOT_IMPLEMENTED   # .vdb files need OpenVDB; density data goes in through b200pt_add_density_grid_to_volume
    assert L.b200pt_add_density_grid_to_volume(None, 0, None) == pt.ERR_WRONG_ARGUMENTS
    buf = np.zeros(16, np.float32); u = np.zeros(4, np.uint32)
    assert L.b200pt_miss_query(None, 1, buf.ctypes.data, u.ctypes.data, buf.ctypes.data, buf.ctypes.data) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_miss_query(None, 1, None, u.ctypes.data, buf.ctypes.data, buf.ctypes.data) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_miss_query(None, 1, buf.ctypes.data, None, buf.ctypes.data, buf.ctypes.data) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_miss_query(None, 1, buf.ctypes.data, u.ctypes.data, None, buf.ctypes.data) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_miss_query(None, 1, buf.ctypes.data, u.ctypes.data, buf.ctypes.data, None) == pt.ERR_WRONG_ARGUMENTS
    m = C.c_uint32()
    assert L.b200pt_bounce_query(None, 1, buf.ctypes.data, 0, buf.ctypes.data, C.byref(m)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_bounce_query(None, 1, None, 0, buf.ctypes.data, C.byref(m)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_bounce_query(None, 1, buf.ctypes.data, 0, None, C.byref(m)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_bounce_query(None, 1, buf.ctypes.data, 0, buf.ctypes.data, None) == pt.ERR_WRONG_ARGUMENTS
    w, h, p = C.c_uint32(), C.c_uint32(), C.c_void_p()
    assert L.b200pt_decode_image_file(b"/nonexistent.png", C.byref(w), C.byref(h), C.byref(p)) == pt.ERR_INIT_FAILED


def test_default_config_matches_reference_defaults():
    c = pt.default_config()                      # PathTracer/PathTracer.h:197-233
    assert (c.SamplesPerFrame, c.MaxSamplesAccumulated, c.MaxDepth, c.MaxLuminance, c.FocusDistance, c.DepthOfFieldStrength) == (1, 5000, 200, 500.0, 1.0, 0.0)
    assert (c.EnableSkyMIS, c.EnableMeshMIS, c.ShowEnvMapDirectly, c.UseOnlyGeometryNormals, c.UseEnergyCompensation, c.FurnaceTestMode) == (1, 1, 1, 0, 1, 0)
    assert (c.SkyIntensity, c.ScreenChunkCount, c.EmissiveMeshSamplingPDFBias) == (1.0, 1, 0.0)
    o = orc.default_config()
    assert (o.SampleCount, o.MaxDepth, o.MaxLuminance) == (c.SamplesPerFrame, c.MaxDepth, c.MaxLuminance)
    assert C.sizeof(pt.Material) == 112 and C.sizeof(pt.Instance) == 72


def test_png_roundtrip_and_decoder_vs_pil(tmp_path):
    from PIL import Image
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (37, 53, 4), dtype=np.uint8)
    p = str(tmp_path / "a.png")
    pt.write_png(p, img)                                       # Editor::SaveToFile path
    assert np.array_equal(np.asarray(Image.open(p).convert("RGBA")), img)
    assert np.array_equal(pt.decode_image(p), img)
    # PIL-written variants: RGB, grey, palette, 16-bit, grey+alpha
    for mode, arr in [("RGB", img[..., :3]), ("L", img[..., 0]), ("LA", img[..., :2])]:
        q = str(tmp_path / f"{mode}.png"); Image.fromarray(arr, mode).save(q)
        assert np.array_equal(pt.decode_image(q), np.asarray(Image.open(q).convert("RGBA")))
    q = str(tmp_path / "pal.png"); Image.fromarray(img[..., :3], "RGB").quantize(17).save(q)
    assert np.array_equal(pt.decode_image(q), np.asarray(Image.open(q).convert("RGBA")))
    q = str(tmp_path / "i16.png"); Image.fromarray((img[..., 0].astype(np.uint16) << 8) | 7).save(q)     # uint16 -> mode "I;16"
    assert np.array_equal(pt.decode_image(q)[..., 0], img[..., 0])          # 16 -> 8 keeps the high byte


def test_jpeg_decoder_close_to_libjpeg(tmp_path):
    from PIL import Image
    rng = np.random.default_rng(1)
    yy, xx = np.mgrid[0:97, 0:131]
    base = np.stack([128 + 100 * np.sin(xx / 17.0), 128 + 100 * np.cos(yy / 11.0), 128 + 60 * np.sin((xx + yy) / 23.0)], -1)
    img = np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)
    for sub, name in [(2, "420"), (0, "444"), (1, "422")]:
        q = str(tmp_path / f"j{name}.jpg"); Image.fromarray(img, "RGB").save(q, quality=92, subsampling=sub)
        mine = pt.decode_image(q).astype(int); ref = np.asarray(Image.open(q).convert("RGBA")).astype(int)
        assert mine.shape == ref.shape
        d = np.abs(mine - ref)
        assert d.max() <= 6 and d.mean() < 0.8, (name, d.max(), d.mean())   # different IDCT / up-sampling rounding only
    q = str(tmp_path / "grey.jpg"); Image.fromarray(img[..., 0], "L").save(q, quality=90)
    assert np.abs(pt.decode_image(q).astype(int) - np.asarray(Image.open(q).convert("RGBA")).astype(int)).max() <= 2


def test_decoders_on_shipped_assets():
    """The shipped textures (stored verbatim) against PIL, and meadow_2_4k.hdr through RLE scanlines copied byte for byte from it, the brightest
    one included (tests/golden/make_golden.py; the whole map decodes to 4096 x 2048 with a maximum of 159744, SURVEY 8c)."""
    from PIL import Image
    for f in ("VikingRoom.png", "BreakfastRoom/tiles.png"):
        assert np.array_equal(pt.decode_image(os.path.join(util.ASSETS, f)), np.asarray(Image.open(os.path.join(util.ASSETS, f)).convert("RGBA")))
    f = os.path.join(util.ASSETS, "BreakfastRoom/picture3.jpg")
    d = np.abs(pt.decode_image(f).astype(int) - np.asarray(Image.open(f).convert("RGBA")).astype(int))
    assert d.max() <= 8 and d.mean() < 1.0
    meta = json.load(open(os.path.join(util.ASSETS, "assets.json")))["meadow_2_4k.hdr"]
    f = os.path.join(util.ASSETS, "meadow_rows.hdr")
    hdr = pt.decode_hdr(f)
    assert hdr.shape == (len(meta["rows"]), 4096, 4) and hdr[..., :3].max() == 159744.0 and np.all(hdr[..., 3] == 1.0)
    assert np.array_equal(hdr, orc.load_hdr(f))


def test_hdr_decoder(tmp_path):
    rng = np.random.default_rng(2)
    rgb = (np.exp(rng.normal(0, 2, (9, 40, 3))) * (rng.random((9, 40, 1)) > 0.1)).astype(np.float32)
    rgb[:, 10:30] = rgb[:, 10:11]                                  # runs
    p = str(tmp_path / "t.hdr"); enc = util.write_rgbe(p, rgb)
    got = pt.decode_hdr(p)
    exp = np.ones((9, 40, 4), np.float32)
    exp[..., :3] = enc[..., :3].astype(np.float32) * np.where(enc[..., 3:] != 0, np.ldexp(np.float32(1.0), enc[..., 3:].astype(int) - 136), 0).astype(np.float32)
    assert np.array_equal(got, exp) and np.array_equal(got, orc.load_hdr(p))


def test_env_alias_table_bit_exact_vs_oracle():
    hot = np.ones((19, 37, 4), np.float32); hot[..., :3] = 0.0; hot[0, 0, :3] = (50.0, 40.0, 30.0)      # one hot texel on the seam and the pole
    half = gltf_ref.synthetic_env(37, 19, 9); half[19 // 2:, :, :3] = 0.0
    const = np.ones((19, 37, 4), np.float32); const[..., :3] = 0.7
    maps = [gltf_ref.synthetic_env(w, h, seed) for seed, (w, h) in [(3, (64, 32)), (4, (128, 64)), (5, (33, 17)), (6, (37, 19)), (7, (37, 1)), (8, (1, 19))]]
    maps += [hot, half, const, gltf_ref.synthetic_env(4096, 2048, seed=3, sun=150000.0)]   # the last: the map bench.py renders with
    for raw in maps:
        a_env, a_alias, a_sum = orc.build_env_alias(raw)
        b_env, b_alias, b_sum = pt.build_env_alias(raw)
        assert np.array_equal(a_env, b_env) and np.array_equal(a_alias, b_alias) and np.float32(a_sum) == np.float32(b_sum)
    z = np.load(os.path.join(util.GOLDEN, "env_alias_kat.npz"))
    env2, alias2, total2 = pt.build_env_alias(z["env"])
    assert np.array_equal(env2, z["env_pdf"]) and np.array_equal(alias2.view(np.uint32).reshape(-1, 2), z["alias"])


def test_camera_round_trip_bit_exact_vs_oracle():
    for name in ("cornell_box", "cornell_box_glass", "viking_room", "breakfast_room"):
        sc = util.scene_dict(name)
        a = orc.camera_from_view(sc["camera_view"], sc["aspect"]); b = pt.camera_from_view(sc["camera_view"], sc["aspect"])
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    vi, pi = pt.camera_from_view(util.scene_dict("cornell_box")["camera_view"], 16 / 9)
    # Q2: 45 degree vertical fov regardless of the glTF yfov: 1/P11 = tan(22.5 deg)
    assert abs(pi[5] - np.tan(np.radians(22.5))) < 1e-6 and abs(pi[0] - 16 / 9 * np.tan(np.radians(22.5))) < 1e-6


def test_bloom_mips_and_partition_helpers():
    assert pt.bloom_mip_sizes(3840, 2160) == orc.bloom_mip_sizes(3840, 2160)
    assert pt.bloom_mip_sizes(1920, 1080) == orc.bloom_mip_sizes(1920, 1080)
    H = 1080
    for world in (1, 2, 4, 8):
        rows = [pt.partition_rows(H, r, world, 16) for r in range(world)]
        allr = np.sort(np.concatenate(rows))
        assert np.array_equal(allr, np.arange(H))                       # disjoint cover
        assert max(len(r) for r in rows) - min(len(r) for r in rows) <= 16
        for r in range(world):
            assert np.all((rows[r] // 16) % world == r)


def _compare_loader(path):
    a = gltf_ref.load_scene(path); b = pt.load_gltf(path)
    assert len(a["meshes"]) == len(b["meshes"]) and len(a["instances"]) == len(b["instances"]) and len(a["textures"]) == len(b["textures"])
    for (va, ia), (vb, ib) in zip(a["meshes"], b["meshes"]):
        assert np.array_equal(ia, ib)
        assert np.array_equal(va["pos"], vb["pos"]) and np.array_equal(va["uv"], vb["uv"])
        assert np.allclose(va["nrm"], vb["nrm"], rtol=0, atol=1.2e-7, equal_nan=True)
    assert np.array_equal(np.frombuffer(a["materials"].tobytes(), np.uint8), b["materials_bytes"])
    for ta, tb in zip(a["textures"], b["textures"]):
        assert ta.shape == tb.shape
        d = np.abs(ta.astype(int) - tb.astype(int)); assert d.max() <= 8          # JPEG only; PNG is exact
        if ta.shape[0] == 1 or path.endswith("VikingRoom.gltf"): assert d.max() == 0
    for (xa, ma, ka), (xb, mb, kb) in zip(a["instances"], b["instances"]):
        assert (ma, ka) == (mb, kb) and np.allclose(xa, xb, rtol=1e-6, atol=1e-6)
    assert np.allclose(a["camera_view"], b["camera_view"], rtol=1e-6, atol=1e-6) and abs(float(a["aspect"]) - float(b["aspect"])) < 1e-7


@pytest.mark.parametrize("name", ["CornellBox", "CornellBoxGlass", "VikingRoom"])
def test_cpp_gltf_loader_matches_oracle_loader_on_shipped_scenes(name):
    _compare_loader(os.path.join(util.ASSETS, name + ".gltf"))


def test_cpp_gltf_loader_on_a_synthetic_scene(tmp_path):
    """Self-authored glTF exercising matrices, TRS nesting, all material extensions, all texture slots, u8/u16/u32 indices."""
    p = util.write_synthetic_gltf(tmp_path)
    _compare_loader(p)
    b = pt.load_gltf(p)
    m = np.frombuffer(b["materials_bytes"].tobytes(), gltf_ref.MATERIAL_DTYPE)
    assert len(m) == 3 and np.allclose(m["EmissiveColor"][0], [3.75, 1.875, 7.5]) and m["Metallic"][1] == 1.0 and m["IOR"][1] == 1.5   # default material appended last
    assert m["RoughnessTextureIndex"][0] == m["MetallicTextureIndex"][0] and b["textures"][m["RoughnessTextureIndex"][0]].shape == (5, 7, 1)   # Q8
    assert len(b["instances"]) == 3 and abs(float(b["aspect"]) - 1.5) < 1e-7
    # Y flip: det of the instance transform is negative (SURVEY Appendix A)
    assert np.linalg.det(b["instances"][2][0].reshape(4, 4).T[:3, :3]) < 0


def _random_bvh2(n_leaves, rng, chain=False):
    """A random binary hierarchy in the product's 64-B node layout: leaves are references ~((first << 2) | (count - 1))."""
    from vpt_b200 import binding as B
    boxes = rng.random((n_leaves, 2, 3)).astype(np.float32); boxes[:, 1] = boxes[:, 0] + 0.05 * rng.random((n_leaves, 3)).astype(np.float32)
    refs = [~((4 * i << 2) | int(rng.integers(0, 4))) for i in range(n_leaves)]
    nodes = np.zeros(n_leaves - 1, B.BVH2_DTYPE)
    box_of = {}
    counter = [0]

    def build(lo, hi):                                   # leaves [lo, hi) -> (child ref, box)
        if hi - lo == 1:
            return refs[lo], boxes[lo]
        idx = counter[0]; counter[0] += 1
        mid = lo + 1 if chain else int(rng.integers(lo + 1, hi))
        ca, ba = build(lo, mid); cb, bb = build(mid, hi)
        nodes[idx]["lo0"], nodes[idx]["hi0"], nodes[idx]["lo1"], nodes[idx]["hi1"] = ba[0], ba[1], bb[0], bb[1]
        nodes[idx]["c0"], nodes[idx]["c1"] = ca, cb
        bx = np.stack([np.minimum(ba[0], bb[0]), np.maximum(ba[1], bb[1])])
        box_of[idx] = bx
        return idx, bx

    import sys
    sys.setrecursionlimit(10000)
    build(0, n_leaves)
    return nodes, refs


@pytest.mark.parametrize("n_leaves,chain", [(2, False), (3, False), (9, False), (1000, False), (40, True)])
def test_bvh4_collapse_preserves_leaves_and_boxes(n_leaves, chain):
    """Host half of the acceleration-structure build (lbvh.cu: bvh4_collapse_host): every BVH2 leaf reference appears exactly once in
    the BVH4, every child box is the box its BVH2 parent stored for it, the layout is breadth-first and the reported depth is exact."""
    from vpt_b200 import binding as B
    rng = np.random.default_rng(n_leaves)
    nodes2, refs = _random_bvh2(n_leaves, rng, chain)
    box2 = {}                                            # child ref -> box as stored in its BVH2 parent
    for n in nodes2:
        box2[int(n["c0"])] = (n["lo0"].copy(), n["hi0"].copy()); box2[int(n["c1"])] = (n["lo1"].copy(), n["hi1"].copy())
    nodes4, depth = B.bvh4_collapse(nodes2, 0)
    assert 1 <= len(nodes4) <= len(nodes2)
    seen_leaves, depth_of, max_d = [], {0: 1}, 1
    inner2_of = {0: 0}                                   # BVH4 node -> BVH2 node it was made from (reconstructed through the boxes)
    for i, n in enumerate(nodes4):
        kids = [int(c) for c in n["child"]]
        used = [k for k in range(4) if kids[k] != B.BVH4_EMPTY]
        assert len(used) >= 2 and used == list(range(len(used)))          # slots are filled from the front
        for k in range(4):
            lo = np.array([n["lox"][k], n["loy"][k], n["loz"][k]]); hi = np.array([n["hix"][k], n["hiy"][k], n["hiz"][k]])
            if k not in used:
                assert np.all(lo == np.float32(3.0e38)) and np.all(hi == np.float32(3.0e38))
                continue
            c = kids[k]
            if c < 0:
                seen_leaves.append(c)
                blo, bhi = box2[c]
                assert np.array_equal(lo, blo) and np.array_equal(hi, bhi)
            else:
                assert i < c < len(nodes4)                                   # breadth-first: children come later
                depth_of[c] = depth_of[i] + 1; max_d = max(max_d, depth_of[c])
                # an inner child's box must be one of the BVH2 inner-node boxes
                assert any(np.array_equal(lo, b[0]) and np.array_equal(hi, b[1]) for r, b in box2.items() if r >= 0)
        if len(used) < 4:
            assert all(kids[k] < 0 for k in used)                            # a node stops short of 4 slots only when all are leaves
    assert sorted(seen_leaves) == sorted(refs)
    assert depth == max_d
    if chain: assert depth <= (n_leaves + 1) // 2 + 1                        # each level absorbs at least two BVH2 levels of a chain... or one + leaf


def test_bvh4_collapse_rejects_bad_arguments_and_leaf_root():
    from vpt_b200 import binding as B
    rng = np.random.default_rng(1)
    nodes2, _ = _random_bvh2(4, rng)
    n4, d = B.bvh4_collapse(nodes2, -5)                   # leaf root: nothing to collapse
    assert len(n4) == 0 and d == 0
    with pytest.raises(B.B200ptError):
        B.bvh4_collapse(nodes2, 99)
    # not a tree: a child index outside the array, a cycle -> zero nodes, no crash / endless loop
    bad = nodes2.copy(); bad[0]["c0"] = 1000
    assert len(B.bvh4_collapse(bad, 0)[0]) == 0
    cyc = nodes2.copy(); cyc[1]["c0"] = 0
    assert len(B.bvh4_collapse(cyc, 0)[0]) == 0


def _bvh2_leaf_sets(nodes, root=0):
    """node index -> (set of leaf refs beneath child0, child1), plus every child box; iterative post-order."""
    under = {}
    order, stack = [], [root]
    while stack:
        n = stack.pop(); order.append(n)
        for c in (int(nodes[n]["c0"]), int(nodes[n]["c1"])):
            if c >= 0: stack.append(c)
    for n in reversed(order):
        sides = []
        for c in (int(nodes[n]["c0"]), int(nodes[n]["c1"])):
            sides.append({c} if c < 0 else under[c][0] | under[c][1])
        under[n] = sides
    return under, order


@pytest.mark.parametrize("n_leaves,chain", [(3, False), (4, False), (64, False), (3000, False), (60, True)])
def test_bvh2_reinsert_keeps_leaves_and_lowers_the_cost(n_leaves, chain):
    """Third opt-in level (lbvh.cu: bvh2_reinsert_host): same leaf references with the same boxes, every child box the exact union of the
    leaf boxes beneath it, depth-first layout with root 0, exact depth, surface-area cost never worse -- starting from a random tree and
    from the binned-SAH tree (little left to find on uniformly scattered boxes; 11 % on BreakfastRoom)."""
    from vpt_b200 import binding as B
    rng = np.random.default_rng(500 + n_leaves)
    nodes2, refs = _random_bvh2(n_leaves, rng, chain)
    leaf_box = {}
    for n in nodes2:
        for c, lo, hi in ((int(n["c0"]), n["lo0"], n["hi0"]), (int(n["c1"]), n["lo1"], n["hi1"])):
            if c < 0: leaf_box[c] = (lo.copy(), hi.copy())
    sah_tree = B.bvh2_sah_rebuild(nodes2, 0)[0]
    for start, passes, frac in ((nodes2, 2, 0.5), (sah_tree, 3, 0.25), (nodes2, 0, 0.5)):
        out, depth, (c0, c1) = B.bvh2_reinsert(start, 0, passes, frac)
        assert len(out) == n_leaves - 1
        under, order = _bvh2_leaf_sets(out, 0)
        assert sorted(order) == list(range(len(out)))
        assert sorted(under[0][0] | under[0][1]) == sorted(refs) and not (under[0][0] & under[0][1])
        dep = {0: 1}
        for n in order:
            for k, c in enumerate((int(out[n]["c0"]), int(out[n]["c1"]))):
                lo, hi = (out[n]["lo1"], out[n]["hi1"]) if k else (out[n]["lo0"], out[n]["hi0"])
                boxes = [leaf_box[r] for r in under[n][k]]
                assert np.array_equal(lo, np.min([b[0] for b in boxes], axis=0)) and np.array_equal(hi, np.max([b[1] for b in boxes], axis=0))
                if c >= 0:
                    assert c > n; dep[c] = dep[n] + 1
            if int(out[n]["c0"]) >= 0: assert int(out[n]["c0"]) == n + 1
        assert depth == max(dep.values())
        assert c1 <= c0 * (1.0 + 1e-5)
        if passes == 0: assert abs(c1 - c0) <= 1e-5 * c0                         # no pass: the tree comes back re-laid-out, cost unchanged
        if n_leaves >= 3000 and start is nodes2 and passes: assert c1 < 0.5 * c0
    with pytest.raises(B.B200ptError):
        B.bvh2_reinsert(nodes2, 0, passes=-1)
    with pytest.raises(B.B200ptError):
        B.bvh2_reinsert(nodes2, 0, fraction=1.5)
    bad = nodes2.copy(); bad[0]["c1"] = 10 ** 6                                  # child index outside the array
    assert len(B.bvh2_reinsert(bad, 0)[0]) == 0
    if n_leaves >= 4:
        cyc = nodes2.copy(); cyc[1]["c0"] = 0                                      # a cycle
        assert len(B.bvh2_reinsert(cyc, 0)[0]) == 0


@pytest.mark.parametrize("n_leaves,chain", [(2, False), (3, False), (64, False), (3000, False), (60, True)])
def test_bvh2_sah_rebuild_keeps_leaves_and_tightens_the_tree(n_leaves, chain):
    """Opt-in tree-quality pass (lbvh.cu: bvh2_sah_rebuild_host): same leaf references with the same boxes, every child box the exact
    union of the leaf boxes beneath it, depth-first layout with root 0, exact depth, and a surface-area cost that does not get worse
    (random input trees: far better)."""
    from vpt_b200 import binding as B
    rng = np.random.default_rng(100 + n_leaves)
    nodes2, refs = _random_bvh2(n_leaves, rng, chain)
    leaf_box = {}
    for n in nodes2:
        for c, lo, hi in ((int(n["c0"]), n["lo0"], n["hi0"]), (int(n["c1"]), n["lo1"], n["hi1"])):
            if c < 0: leaf_box[c] = (lo.copy(), hi.copy())
    out, depth, (sah0, sah1) = B.bvh2_sah_rebuild(nodes2, 0)
    assert len(out) == n_leaves - 1
    under, order = _bvh2_leaf_sets(out, 0)
    assert sorted(order) == list(range(len(out)))                               # every node reachable exactly once
    assert sorted(under[0][0] | under[0][1]) == sorted(refs) and not (under[0][0] & under[0][1])
    dep = {0: 1}
    for n in order:                                                             # pre-order: parents before children
        for k, c in enumerate((int(out[n]["c0"]), int(out[n]["c1"]))):
            lo, hi = (out[n]["lo1"], out[n]["hi1"]) if k else (out[n]["lo0"], out[n]["hi0"])
            boxes = [leaf_box[r] for r in under[n][k]]
            assert np.array_equal(lo, np.min([b[0] for b in boxes], axis=0)) and np.array_equal(hi, np.max([b[1] for b in boxes], axis=0))
            if c >= 0:
                assert c > n                                                    # children come later in the array
                dep[c] = dep[n] + 1
        if int(out[n]["c0"]) >= 0: assert int(out[n]["c0"]) == n + 1            # depth-first: the left child follows its parent
    assert depth == max(dep.values())
    assert sah1 <= sah0 * (1.0 + 1e-6)
    if n_leaves >= 64: assert sah1 < 0.6 * sah0 and depth <= 4 * int(np.ceil(np.log2(n_leaves)))
    # idempotent in cost: rebuilding the rebuilt tree does not change its cost
    out2, depth2, (s0, s1) = B.bvh2_sah_rebuild(out, 0)
    assert abs(s0 - sah1) <= 1e-9 * max(1.0, sah1) and s1 <= s0 * (1.0 + 1e-6)


def test_bvh2_sah_rebuild_rejects_bad_input():
    from vpt_b200 import binding as B
    rng = np.random.default_rng(2)
    nodes2, _ = _random_bvh2(5, rng)
    assert len(B.bvh2_sah_rebuild(nodes2, -3)[0]) == 0                            # leaf root
    with pytest.raises(B.B200ptError):
        B.bvh2_sah_rebuild(nodes2, 77)
    bad = nodes2.copy(); bad[0]["c1"] = 1000
    assert len(B.bvh2_sah_rebuild(bad, 0)[0]) == 0
    cyc = nodes2.copy(); cyc[1]["c0"] = 0
    assert len(B.bvh2_sah_rebuild(cyc, 0)[0]) == 0


@pytest.mark.parametrize("n,tc", [(5, 1.0), (6, 1.0), (257, 1.0), (5000, 1.0), (5000, 3.0)])
def test_bvh2_sah_build_from_reference_boxes(n, tc):
    """Second opt-in level (lbvh.cu: bvh2_sah_build_host): perm is a permutation, the leaves tile [0, n) with <= 4 slots each, child boxes
    contain the padded union of the reference boxes beneath them, layout is depth-first, and a ray walk through the tree finds the
    same closest hits as brute force over all triangles."""
    import sys as _sys
    _sys.path.insert(0, os.path.join(util.ROOT, "profiles"))
    import bvh_lab
    from vpt_b200 import binding as B
    rng = np.random.default_rng(n)
    ctr = rng.random((n, 1, 3)).astype(np.float32) * 4 - 2
    tri = (ctr + 0.15 * (rng.random((n, 3, 3)).astype(np.float32) - 0.5)).astype(np.float32)
    rb = np.concatenate([tri.min(1), tri.max(1)], 1)
    nodes, perm, depth, cost = B.bvh2_sah_build(rb, tc)
    assert sorted(perm.tolist()) == list(range(n)) and 1 <= len(nodes) <= n - 1 and cost > 0
    ext = np.abs(rb).max(); pabs = np.float32(2e-6) * ext
    covered = np.zeros(n, np.int32); dep = {0: 1}
    under = {}
    for i in range(len(nodes) - 1, -1, -1):                                      # children come later: a reverse sweep is a post-order
        sides = []
        for k, c in enumerate((int(nodes[i]["c0"]), int(nodes[i]["c1"]))):
            if c < 0:
                r = ~c; first, cnt = r >> 2, (r & 3) + 1
                assert cnt <= 4 and first + cnt <= n
                covered[first:first + cnt] += 1
                lo, hi = rb[perm[first:first + cnt], :3].min(0), rb[perm[first:first + cnt], 3:].max(0)
            else:
                assert i < c < len(nodes)
                lo, hi = under[c]
            blo, bhi = (nodes[i]["lo1"], nodes[i]["hi1"]) if k else (nodes[i]["lo0"], nodes[i]["hi0"])
            pad = np.float32(4e-7) * np.maximum(np.abs(lo), np.abs(hi)) + pabs
            assert np.all(blo <= lo - 0.5 * pad) and np.all(bhi >= hi + 0.5 * pad) and np.all(blo >= lo - 2 * pad) and np.all(bhi <= hi + 2 * pad)
            sides.append((lo, hi))
        under[i] = (np.minimum(sides[0][0], sides[1][0]), np.maximum(sides[0][1], sides[1][1]))
    assert np.all(covered == 1)
    for i in range(len(nodes)):
        for c in (int(nodes[i]["c0"]), int(nodes[i]["c1"])):
            if c >= 0: dep[c] = dep[i] + 1
        if int(nodes[i]["c0"]) >= 0: assert int(nodes[i]["c0"]) == i + 1
    assert depth == max(dep.values()) and depth <= 6 * int(np.ceil(np.log2(n))) + 2
    # identical closest hits: tree walk vs brute force
    R = 400
    O = (rng.random((R, 3)) * 6 - 3); D = tri[rng.integers(0, n, R)].mean(1) + 0.02 * rng.normal(size=(R, 3)) - O    # aimed at triangles, so most rays hit
    D /= np.linalg.norm(D, axis=1, keepdims=True)
    t_tree, _, _ = bvh_lab.traverse(nodes, tri[perm], O, D)
    t_brute = np.full(R, np.inf)
    E1, E2 = (tri[:, 1] - tri[:, 0]).astype(np.float64), (tri[:, 2] - tri[:, 0]).astype(np.float64); A = tri[:, 0].astype(np.float64)
    for r in range(R):
        p = np.cross(D[r], E2); det = (E1 * p).sum(1); ok = np.abs(det) > 1e-30; idet = 1.0 / np.where(ok, det, 1.0)
        sv = O[r] - A; u = (sv * p).sum(1) * idet; q = np.cross(sv, E1); v = (q * D[r]).sum(1) * idet; tt = (E2 * q).sum(1) * idet
        hit = ok & (u >= 0) & (v >= 0) & (u + v <= 1) & (tt > 1e-6)
        if hit.any(): t_brute[r] = tt[hit].min()
    assert np.array_equal(np.isfinite(t_tree), np.isfinite(t_brute)) and np.allclose(t_tree[np.isfinite(t_tree)], t_brute[np.isfinite(t_brute)], rtol=1e-12)
    assert np.isfinite(t_brute).sum() > R // 4


def test_bvh2_sah_build_rejects_degenerate_input():
    from vpt_b200 import binding as B
    rb = np.zeros((4, 6), np.float32)
    assert len(B.bvh2_sah_build(rb)[0]) == 0                                      # one leaf: the caller keeps what it has
    rb = np.zeros((9, 6), np.float32); rb[:, 3:] = 1.0                            # identical boxes: median splits, still a valid tree
    nodes, perm, depth, _ = B.bvh2_sah_build(rb)
    assert len(nodes) >= 2 and sorted(perm.tolist()) == list(range(9))
    bad = rb.copy(); bad[3, 0] = np.nan
    assert len(B.bvh2_sah_build(bad)[0]) == 0
    inv = rb.copy(); inv[2, 3] = -5.0
    assert len(B.bvh2_sah_build(inv)[0]) == 0


def test_bvh2_sah_rebuild_is_independent_of_the_thread_count(monkeypatch):
    """The inner-node rebuild forks its large right subtrees onto host threads (node indices are known in advance: k leaves -> k - 1
    nodes); the emitted array must not depend on how many threads took part."""
    from vpt_b200 import binding as B
    rng = np.random.default_rng(77)
    nodes2, _ = _random_bvh2(40000, rng)
    outs = []
    for threads in ("1", "2", "5", "64"):
        monkeypatch.setenv("B200PT_HOST_THREADS", threads)
        out, depth, (c0, c1) = B.bvh2_sah_rebuild(nodes2, 0)
        outs.append((out.tobytes(), depth, c1))
    for o in outs[1:]:
        assert o[0] == outs[0][0] and o[1] == outs[0][1] and o[2] == outs[0][2]
    # the full build (leaves re-formed: node blocks are compacted afterwards) as well
    ctr = rng.random((60000, 3)).astype(np.float32); ext = (0.01 * rng.random((60000, 3))).astype(np.float32)
    rb = np.concatenate([ctr - ext, ctr + ext], 1)
    outs = []
    for threads in ("1", "3", "16"):
        monkeypatch.setenv("B200PT_HOST_THREADS", threads)
        nodes, perm, depth, cost = B.bvh2_sah_build(rb, 1.0)
        outs.append((nodes.tobytes(), perm.tobytes(), depth, cost))
    assert outs[1] == outs[0] and outs[2] == outs[0]


def test_refine_sah_plumbing_with_caller_reference_boxes(tmp_path):
    """lbvh_refine_sah (the device-touching half of the opt-in tree passes) run on host arrays, with the reference boxes passed by the caller
    (null outside modes 2 / 3): tests/native/refine_plumbing.cpp replaces the three CUDA copy calls by memcpy shims and cudaFree by a no-op
    (the tree's owners wrap host vectors), then checks for modes 0..5 that every ray finds the same closest triangle as brute force, that
    tri_slot survives the slot permutation of modes 2 / 3, root / max_depth bookkeeping and that a costlier tree is never uploaded."""
    import shutil, subprocess
    obj = os.path.join(util.ROOT, "vulkan-path-tracer_b200", "build", "lbvh.o")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(obj) or not os.path.exists(nvcc): pytest.skip("needs nvcc and the built lbvh.o")
    exe = str(tmp_path / "refine_plumbing")
    cmd = [nvcc, "--cudart", "shared", "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-I" + os.path.join(util.ROOT, "vulkan-path-tracer_b200", "csrc"),
           "-I" + os.path.join(util.ROOT, "include"), os.path.join(util.ROOT, "tests", "native", "refine_plumbing.cpp"), obj, "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-2000:]
    assert r.stdout.count(": ok,") == 36                                          # 6 scenes x modes 0..5


def test_atmosphere_block_defaults_match_the_reference_members():
    """b200pt_atmosphere = the twelve atmosphere members of PathTracer.h:221-232 behind their setters / getters (:129-144,170-181)."""
    import ctypes as C
    L = pt.lib()
    a = pt.Atmosphere()
    assert C.sizeof(a) == 88
    assert L.b200pt_default_atmosphere(C.byref(a)) == pt.OK
    assert a.Enable == 0 and tuple(a.PlanetPosition) == (0.0, np.float32(6360e3 + 1000.0), 0.0) and a.PlanetRadius == np.float32(6360e3)
    assert a.AtmosphereHeight == 100e3 and tuple(a.SunColor) == (1.0, np.float32(0.956), np.float32(0.88))
    assert (a.RayleighDensityFalloff, a.MieDensityFalloff, a.OzoneDensityFalloff, a.OzonePeak) == (8000.0, 1200.0, 5000.0, 22000.0)
    for v in (a.RayleighScatteringCoefficientMultiplier, a.MieScatteringCoefficientMultiplier, a.OzoneAbsorptionCoefficientMultiplier): assert tuple(v) == (1.0, 1.0, 1.0)
    assert L.b200pt_default_atmosphere(None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_set_atmosphere(None, C.byref(a)) == pt.ERR_WRONG_ARGUMENTS and L.b200pt_get_total_counts(None, None, None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_remove_density_data_from_volume(None, 0) == pt.ERR_WRONG_ARGUMENTS


def test_volume_struct_and_defaults_without_gpu():
    """b200pt_volume mirrors PathTracer::Volume (PT/PathTracer.h:36-70): layout and defaults are checked on the CPU."""
    import ctypes as C
    from vpt_b200 import binding as B
    assert C.sizeof(B.Volume) == 148 and C.sizeof(B.DensityGrid) == 80
    v = B.PathTracer.make_volume()
    assert list(v.CornerMin) == [-1.0] * 3 and list(v.CornerMax) == [1.0] * 3 and list(v.Position) == [0.0] * 3 and list(v.Scale) == [1.0] * 3
    assert all(abs(c - 0.8) < 1e-7 for c in v.Color) and list(v.EmissiveColor) == [0.0] * 3 and list(v.TemperatureColor) == [1.0, 0.5, 0.0]
    assert (v.Density, v.Anisotropy, v.Alpha, v.DropletSize, v.DensityDataIndex, v.MaxDensityInTheGrid) == (1.0, 0.0, 1.0, 20.0, -1, 0.0)
    assert (v.UseBlackbody, v.HasTemperatureData, v.TemperatureGamma, v.TemperatureScale, v.EmissiveColorGamma, v.KelvinMin, v.KelvinMax) == (1, 0, 1.0, 1.0, 1.0, 500, 8000)
    assert v.ApproximatedScatteringForClouds == 0 and abs(v.ApproximatedScatteringFalloff - 0.8) < 1e-7 and v.GridSharpness == 1.0
    assert B.lib().b200pt_default_volume(None) == B.ERR_WRONG_ARGUMENTS


def test_density_grid_preparation_equals_the_oracle():
    """The host half of AddDensityDataToVolume (PT/PathTracer.cpp:1391-1452) in csrc/density_grid.cpp against the oracle's restatement, bit for bit:
    MaxDensityInTheGrid, the AABB scaled into [-1, 1], the 32^3 majorants gathered with Y flipped and integer cell arithmetic, and the reference's
    temperature patch (normalised temperature written INTO the density grid wherever it is positive)."""
    from vpt_b200 import binding as B
    from oracle import orc
    rs = np.random.RandomState(11)
    for shape, imin, with_t in (((21, 37, 18), (-9, -20, -7), True), ((64, 40, 70), (3, -50, 10), False), ((5, 3, 2), (0, 0, 0), True)):
        d = rs.rand(*shape).astype(np.float32) ** 3 * 4.0
        d[rs.rand(*shape) < 0.4] = 0.0
        t = (rs.rand(*shape).astype(np.float32) * 900.0 - 200.0) if with_t else None
        if t is not None: t[rs.rand(*shape) < 0.5] = -200.0
        g = orc.prepare_density_grid(d, index_min=imin, temperature=t, voxel_size=0.5, translation=(1.0, -2.0, 0.25))
        vals, maj, cmin, cmax, mx = B.prepare_density_grid(d, index_min=imin, temperature=t, voxel_size=0.5, translation=(1.0, -2.0, 0.25))
        assert mx == g["max_density"] == float(d.max()) and cmin == g["corner_min"] and cmax == g["corner_max"]
        assert np.array_equal(vals.view(np.uint32), g["values"].view(np.uint32)) and np.array_equal(maj.view(np.uint32), g["max_densities"].view(np.uint32))
        assert max(abs(c) for c in cmin + cmax) == 1.0                               # the largest |index coordinate| maps to 1
        if with_t: assert (vals != d).any() and np.all(vals[t <= t.min()] == d[t <= t.min()])   # patched exactly where the normalised temperature is positive
        else: assert np.array_equal(vals, d)
    # a single hot voxel lands in the majorant cell of its FLIPPED row (PathTracer.cpp:1432-1436)
    d = np.zeros((8, 16, 4), np.float32); d[2, 3, 1] = 7.0
    _, maj, _, _, mx = B.prepare_density_grid(d)
    cell = (1 * 32) // 4 + (((16 - 1 - 3) * 32) // 16) * 32 + ((2 * 32) // 8) * 1024
    assert mx == 7.0 and maj[cell] == 1.0 and np.count_nonzero(maj) == 1
    L = B.lib()
    g, keep = B.make_density_grid(np.zeros((2, 2, 2), np.float32))
    out = np.zeros(8, np.float32); m = np.zeros(32768, np.float32); c3 = (C.c_float * 3)(); f = C.c_float()
    args = (out.ctypes.data_as(C.c_void_p), m.ctypes.data_as(C.c_void_p), c3, c3, C.byref(f))
    assert L.b200pt_prepare_density_grid(C.byref(g), *args) == B.ERR_WRONG_ARGUMENTS          # no positive density
    assert L.b200pt_prepare_density_grid(None, *args) == B.ERR_WRONG_ARGUMENTS
    g, keep = B.make_density_grid(np.ones((2, 2, 2), np.float32), voxel_size=0.0)
    assert L.b200pt_prepare_density_grid(C.byref(g), *args) == B.ERR_WRONG_ARGUMENTS


def test_density_grid_preparation_property():
    """Property form of the test above (hypothesis): any bbox shape, origin, temperature presence and explicit temperature range -- the product's host half and
    the oracle's restatement of PathTracer.cpp:1391-1452 agree bit for bit, every majorant dominates the normalised values gathered into its cell, and
    cells no voxel maps to stay 0."""
    from hypothesis import given, settings, strategies as st
    from vpt_b200 import binding as B
    from oracle import orc

    @settings(max_examples=40, deadline=None)
    @given(st.tuples(st.integers(1, 40), st.integers(1, 40), st.integers(1, 40)), st.tuples(st.integers(-60, 60), st.integers(-60, 60), st.integers(-60, 60)),
           st.booleans(), st.integers(0, 2 ** 31 - 1))
    def run(shape, imin, with_t, seed):
        rs = np.random.RandomState(seed)
        d = (rs.rand(*shape).astype(np.float32) * 3.0 + 0.01) * (rs.rand(*shape) > 0.3)
        d.flat[rs.randint(d.size)] = 3.5                                              # at least one positive value
        t = (rs.rand(*shape).astype(np.float32) * 1000.0) if with_t else None
        tr = (50.0, 800.0) if with_t and seed % 2 else None                          # explicit range of the temperature tree's active values, or derived from the array
        g = orc.prepare_density_grid(d, index_min=imin, temperature=t, temperature_range=tr)
        vals, maj, cmin, cmax, mx = B.prepare_density_grid(d, index_min=imin, temperature=t, temperature_range=tr)
        # (a bbox whose every index coordinate is 0 scales by 0 / 0: NaN corners in the reference, PathTracer.cpp:1415-1420, and in both restatements)
        assert mx == g["max_density"] and np.array_equal(np.array(cmin + cmax, np.float32).view(np.uint32), np.array(g["corner_min"] + g["corner_max"], np.float32).view(np.uint32))
        assert np.array_equal(vals.view(np.uint32), g["values"].view(np.uint32)) and np.array_equal(maj.view(np.uint32), g["max_densities"].view(np.uint32))
        nz, ny, nx = shape
        zz, yy, xx = np.mgrid[0:nz, 0:ny, 0:nx]
        cell = (xx * 32) // nx + (((ny - 1 - yy) * 32) // ny) * 32 + ((zz * 32) // nz) * 1024        # array row yy is the loop's y = ny - 1 - yy
        want = np.zeros(32768, np.float32); np.maximum.at(want, cell.ravel(), np.clip(d / np.float32(mx), 0.0, 1.0).astype(np.float32).ravel())
        assert np.array_equal(maj, want)
    run()


def test_cli_renderer_builds_and_fails_loudly_without_a_gpu():
    """b200pt_render (csrc/cli_main.cpp), the headless stand-in for the reference's Editor: built next to the library, prints its usage,
    and -- like every product path -- refuses to run without a CUDA device instead of falling back to anything."""
    import subprocess, torch
    exe = os.path.join(os.path.dirname(pt.LIB_PATH), "b200pt_render")
    assert os.path.exists(exe)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "usage: b200pt_render" in r.stderr and "--atmosphere" in r.stderr and "--volume" in r.stderr
    if not torch.cuda.is_available():
        r = subprocess.run([exe, "--scene", "s.gltf", "--env", "e.hdr", "--luts", "d", "--out", "o.png"], capture_output=True, text=True)
        assert r.returncode != 0 and "no CUDA device" in r.stderr


def test_cpp_gltf_loader_reads_glb_and_base64_buffers(tmp_path):
    """assimp's glTF2 importer (the reference's loader, AssetImporterImpl.cpp:82-97) also reads binary .glb containers and base64 data: URIs
    for geometry buffers.  The same synthetic scene stored three ways must load to identical arrays; embedded TEXTURES are rejected with an
    error (the reference only loads texture files next to the model, :287-328)."""
    import base64, struct
    p = util.write_synthetic_gltf(tmp_path)
    g = json.load(open(p)); blob = (tmp_path / "s.bin").read_bytes()
    ref = pt.load_gltf(p)
    # (a) base64 data URI
    g64 = json.loads(json.dumps(g)); g64["buffers"][0] = {"uri": "data:application/octet-stream;base64," + base64.b64encode(blob).decode(), "byteLength": len(blob)}
    pa = str(tmp_path / "s64.gltf"); open(pa, "w").write(json.dumps(g64))
    # (b) .glb: JSON chunk + BIN chunk, textures stay external
    gb = json.loads(json.dumps(g)); gb["buffers"][0] = {"byteLength": len(blob)}
    jtxt = json.dumps(gb).encode(); jtxt += b" " * (-len(jtxt) % 4); bchunk = blob + b"\0" * (-len(blob) % 4)
    glb = b"glTF" + struct.pack("<II", 2, 12 + 8 + len(jtxt) + 8 + len(bchunk)) + struct.pack("<II", len(jtxt), 0x4E4F534A) + jtxt + struct.pack("<II", len(bchunk), 0x004E4942) + bchunk
    pb = str(tmp_path / "s.glb"); open(pb, "wb").write(glb)
    for q in (pa, pb):
        _compare_loader(q)                                         # C++ loader == oracle-side python loader
        b = pt.load_gltf(q)
        assert len(b["meshes"]) == len(ref["meshes"]) and len(b["instances"]) == len(ref["instances"])
        for (v0, i0), (v1, i1) in zip(ref["meshes"], b["meshes"]):
            assert np.array_equal(v0, v1) and np.array_equal(i0, i1)
        assert np.array_equal(ref["materials_bytes"], b["materials_bytes"])
        for t0, t1 in zip(ref["textures"], b["textures"]): assert np.array_equal(t0, t1)
    # embedded image -> error code, no crash
    ge = json.loads(json.dumps(g)); ge["images"][0] = {"uri": "data:image/png;base64,AAAA"}
    pe = str(tmp_path / "emb.gltf"); open(pe, "w").write(json.dumps(ge))
    with pytest.raises(pt.B200ptError): pt.load_gltf(pe)
    # truncated .glb -> error code
    open(str(tmp_path / "bad.glb"), "wb").write(glb[:40])
    with pytest.raises(pt.B200ptError): pt.load_gltf(str(tmp_path / "bad.glb"))


def _write_png_adam7(path, arr, ctype, depth=8, palette=None, sub_filter=False):
    """Tiny PNG writer with Adam7 interlacing (PIL cannot write interlaced files).  arr: HxWxC uint8 samples (C = channels of ctype; for
    depth < 8, values < 2**depth)."""
    import struct, zlib
    H, W = arr.shape[:2]; C = arr.shape[2]
    def chunk(t, d): return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)
    xs, ys, dx, dy = (0, 4, 0, 2, 0, 1, 0), (0, 0, 4, 0, 2, 0, 1), (8, 8, 4, 4, 2, 2, 1), (8, 8, 8, 4, 4, 2, 2)
    raw = b""
    for p in range(7):
        sub = arr[ys[p]::dy[p], xs[p]::dx[p]]
        if sub.shape[0] == 0 or sub.shape[1] == 0: continue
        for row in sub:
            samples = row.reshape(-1)
            if depth == 8: b = bytes(samples)
            elif depth == 16: b = b"".join(bytes([int(v), 0x5A]) for v in samples)
            else:
                bits = "".join(format(int(v), f"0{depth}b") for v in samples); bits += "0" * (-len(bits) % 8)
                b = bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))
            if sub_filter:
                bpp = max(1, C * depth // 8); f = bytearray(b)
                for i in range(len(b) - 1, bpp - 1, -1): f[i] = (b[i] - b[i - bpp]) & 255
                raw += b"\x01" + bytes(f)
            else:
                raw += b"\x00" + b
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ctype, 0, 0, 1))
    if palette is not None: out += chunk(b"PLTE", bytes(palette.reshape(-1)))
    out += chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b"")
    open(path, "wb").write(out)


def test_png_decoder_reads_adam7_interlaced_files(tmp_path):
    """stb_image (the reference's texture decoder, AssetImporterImpl.cpp:494-545) reads interlaced PNGs; so does ours, for every colour type,
    1..16-bit samples, odd sizes smaller than the 8x8 interlace cell, and filtered scanlines inside the passes."""
    rng = np.random.default_rng(11)
    for (W, H) in ((1, 1), (3, 2), (9, 5), (33, 17)):
        rgba = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
        p = str(tmp_path / "a.png"); _write_png_adam7(p, rgba, 6); assert np.array_equal(pt.decode_image(p), rgba)
        _write_png_adam7(p, rgba, 6, sub_filter=True); assert np.array_equal(pt.decode_image(p), rgba)
        rgb = rgba[..., :3]; _write_png_adam7(p, rgb, 2); got = pt.decode_image(p); assert np.array_equal(got[..., :3], rgb) and np.all(got[..., 3] == 255)
        _write_png_adam7(p, rgba, 6, depth=16); assert np.array_equal(pt.decode_image(p), rgba)      # high byte kept
        ga = rgba[..., :2]; _write_png_adam7(p, ga, 4); got = pt.decode_image(p)
        assert np.array_equal(got[..., 0], ga[..., 0]) and np.array_equal(got[..., 1], ga[..., 0]) and np.array_equal(got[..., 3], ga[..., 1])
        for depth in (1, 2, 4):
            g = rng.integers(0, 2 ** depth, (H, W, 1), dtype=np.uint8); _write_png_adam7(p, g, 0, depth=depth)
            assert np.array_equal(pt.decode_image(p)[..., 0], g[..., 0] * (255 // (2 ** depth - 1)))
            pal = rng.integers(0, 256, (2 ** depth, 3), dtype=np.uint8); _write_png_adam7(p, g, 3, depth=depth, palette=pal)
            assert np.array_equal(pt.decode_image(p)[..., :3], pal[g[..., 0]])


def test_progressive_jpeg_decodes_like_the_baseline_file(tmp_path):
    """stb_image (AssetImporterImpl.cpp:494-545) reads progressive JPEGs (SOF2: spectral selection + successive approximation, ITU T.81
    annex G).  The coefficients of a progressive file equal those of the baseline file made from the same image and quality, so OUR decode of
    both must be bit-identical; against libjpeg only IDCT / up-sampling rounding differs (same bound as the baseline test)."""
    from PIL import Image
    rng = np.random.default_rng(4)
    yy, xx = np.mgrid[0:75, 0:118]
    base = np.stack([128 + 100 * np.sin(xx / 13.0), 128 + 100 * np.cos(yy / 9.0), 128 + 60 * np.sin((xx + yy) / 19.0)], -1)
    img = np.clip(base + rng.normal(0, 8, base.shape), 0, 255).astype(np.uint8)
    for sub, name in [(2, "420"), (0, "444"), (1, "422")]:
        qb = str(tmp_path / f"b{name}.jpg"); qp = str(tmp_path / f"p{name}.jpg")
        Image.fromarray(img, "RGB").save(qb, quality=88, subsampling=sub)
        Image.fromarray(img, "RGB").save(qp, quality=88, subsampling=sub, progressive=True)
        assert b"\xff\xc2" in open(qp, "rb").read() and b"\xff\xc2" not in open(qb, "rb").read()
        mine = pt.decode_image(qp)
        assert np.array_equal(mine, pt.decode_image(qb)), name
        d = np.abs(mine.astype(int) - np.asarray(Image.open(qp).convert("RGBA")).astype(int))
        assert d.max() <= 6 and d.mean() < 0.8, (name, d.max(), d.mean())
    qg = str(tmp_path / "pg.jpg"); Image.fromarray(img[..., 1], "L").save(qg, quality=85, progressive=True)
    assert np.abs(pt.decode_image(qg).astype(int) - np.asarray(Image.open(qg).convert("RGBA")).astype(int)).max() <= 2
    # restart intervals inside progressive scans
    qr = str(tmp_path / "pr.jpg"); Image.fromarray(img, "RGB").save(qr, quality=80, progressive=True, restart_marker_blocks=3)
    d = np.abs(pt.decode_image(qr).astype(int) - np.asarray(Image.open(qr).convert("RGBA")).astype(int))
    assert d.max() <= 6 and d.mean() < 0.8
    # truncated file: error code, no crash
    raw = open(qp, "rb").read(); open(str(tmp_path / "cut.jpg"), "wb").write(raw[:len(raw) // 3])
    try: pt.decode_image(str(tmp_path / "cut.jpg"))
    except pt.B200ptError: pass


def test_gltf_without_normals_gets_assimp_style_face_normals(tmp_path):
    """aiProcess_GenNormals (AssetImporterImpl.cpp:82-97): a primitive without NORMAL gets flat face normals the way assimp 6.0.2 writes them
    (a shared vertex keeps the normal of the last face that uses it).  C++ loader == oracle-side loader, and the values are the expected ones."""
    pos = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [5, 5, 5]], np.float32)        # vertex 4 is referenced by no face
    idx = np.array([0, 1, 2, 0, 3, 1], np.uint16)                                                # faces normal to +z then +y... (0,3,1): (3-0)x(1-0) = z x x = +y
    blob = pos.tobytes() + idx.tobytes()
    (tmp_path / "n.bin").write_bytes(blob)
    g = {"asset": {"version": "2.0"}, "scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0}],
         "meshes": [{"primitives": [{"attributes": {"POSITION": 0}, "indices": 1}]}],
         "accessors": [{"bufferView": 0, "componentType": 5126, "count": 5, "type": "VEC3"}, {"bufferView": 1, "componentType": 5123, "count": 6, "type": "SCALAR"}],
         "bufferViews": [{"buffer": 0, "byteOffset": 0, "byteLength": 60}, {"buffer": 0, "byteOffset": 60, "byteLength": 12}],
         "buffers": [{"uri": "n.bin", "byteLength": len(blob)}]}
    p = str(tmp_path / "n.gltf"); open(p, "w").write(json.dumps(g))
    _compare_loader(p)
    v, i = pt.load_gltf(p)["meshes"][0]
    nrm = np.asarray(v["nrm"], np.float32)
    assert np.allclose(nrm[2], [0, 0, 1]) and np.allclose(nrm[3], [0, 1, 0])                 # only in one face each
    assert np.allclose(nrm[0], [0, 1, 0]) and np.allclose(nrm[1], [0, 1, 0])                 # shared: the LAST face (0,3,1) wins
    assert np.isnan(nrm[4]).all()                                                            # glm::normalize of the zero vector, like the reference


def test_gltf_strips_and_fans_become_triangles(tmp_path):
    """glTF primitive modes 5 / 6: the reference's importer (assimp glTF2) expands strips and fans into faces; same face list in both loaders."""
    pos = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 1, 0]], np.float32)
    idx = np.array([0, 1, 2, 3, 4], np.uint16)
    blob = pos.tobytes() + idx.tobytes() + b"\0\0"
    (tmp_path / "s.bin").write_bytes(blob)
    for mode, want in ((5, [0, 1, 2, 2, 1, 3, 2, 3, 4]), (6, [0, 1, 2, 0, 2, 3, 0, 3, 4])):
        g = {"asset": {"version": "2.0"}, "scene": 0, "scenes": [{"nodes": [0]}], "nodes": [{"mesh": 0}],
             "meshes": [{"primitives": [{"attributes": {"POSITION": 0}, "indices": 1, "mode": mode}]}],
             "accessors": [{"bufferView": 0, "componentType": 5126, "count": 5, "type": "VEC3"}, {"bufferView": 1, "componentType": 5123, "count": 5, "type": "SCALAR"}],
             "bufferViews": [{"buffer": 0, "byteOffset": 0, "byteLength": 60}, {"buffer": 0, "byteOffset": 60, "byteLength": 10}],
             "buffers": [{"uri": "s.bin", "byteLength": len(blob)}]}
        p = str(tmp_path / f"m{mode}.gltf"); open(p, "w").write(json.dumps(g))
        _compare_loader(p)
        assert list(pt.load_gltf(p)["meshes"][0][1]) == want
    g["meshes"][0]["primitives"][0]["mode"] = 1
    p = str(tmp_path / "lines.gltf"); open(p, "w").write(json.dumps(g))
    with pytest.raises(pt.B200ptError): pt.load_gltf(p)


def test_obj_mtl_import(tmp_path):
    """Wavefront OBJ + MTL through the same entry point as glTF (AssetImporter::ImportScene picks the importer by extension): quads and n-gons
    become fans, (v, vt, vn) triples are joined, missing normals are generated per face, uv is flipped, materials follow the keys the reference
    reads (AssetImporterImpl.cpp:353-455) with assimp's OBJ defaults.  C++ loader == oracle-side loader, plus the expected values."""
    from PIL import Image
    rng = np.random.default_rng(8)
    Image.fromarray(rng.integers(0, 256, (4, 6, 3), dtype=np.uint8), "RGB").save(tmp_path / "kd.png")
    Image.fromarray(rng.integers(0, 256, (3, 3, 3), dtype=np.uint8), "RGB").save(tmp_path / "ke.png")
    (tmp_path / "m.mtl").write_text(
        "# materials\nnewmtl red\nKd 0.8 0.1 0.1\nKs 0.5 0.5 0.5\nNi 1.45\nPr 0.3\nPm 0.2\naniso 0.4\nanisor 0.5\nmap_Kd -bm 1.0 kd.png\n"
        "newmtl lamp\nKd 1 1 1\nKe 5 4 3\nmap_Ke ke.png\nmap_bump ignored.png\n\nnewmtl unused\nKd 0 1 0\n")
    (tmp_path / "s.obj").write_text(
        "mtllib m.mtl\no floor\nv 0 0 0\nv 2 0 0\nv 2 0 2\nv 0 0 2\nv 1 1 1\nvt 0 0\nvt 1 0\nvt 1 1\nvt 0 1\nvn 0 1 0\n"
        "f 1/1/1 2/2/1 3/3/1 4/4/1\n"                       # quad with uv + normals, default material
        "usemtl red\nf 1 2 5\nf -4//1 -3//1 -1//1 \\\n  -5//1\n"   # no normals at all -> generated; negative indices + line continuation
        "g lampgroup\nusemtl lamp\nf 3/3 4/4 5/1\n")
    p = str(tmp_path / "s.obj")
    _compare_loader(p)
    b = pt.load_gltf(p)
    m = np.frombuffer(b["materials_bytes"].tobytes(), gltf_ref.MATERIAL_DTYPE)
    assert len(m) == 4                                           # DefaultMaterial + 3 newmtl
    assert np.allclose(m["BaseColor"][0], 0.6) and m["IOR"][0] == 1.0 and m["Metallic"][0] == 0.0 and m["Roughness"][0] == 1.0 and np.all(m["SpecularColor"][0] == 0)
    assert np.allclose(m["BaseColor"][1], [0.8, 0.1, 0.1]) and abs(m["IOR"][1] - 1.45) < 1e-6 and abs(m["Roughness"][1] - 0.3) < 1e-6 and abs(m["Metallic"][1] - 0.2) < 1e-6
    assert abs(m["AnisotropyRotation"][1] - np.degrees(0.5)) < 1e-4 and np.allclose(m["EmissiveColor"][2], [5, 4, 3])
    assert b["textures"][m["BaseColorTextureIndex"][1]].shape == (4, 6, 4) and b["textures"][m["EmissiveTextureIndex"][2]].shape == (3, 3, 4)
    assert b["textures"][m["NormalTextureIndex"][2]].shape == (1, 1, 4)          # map_bump is a height map: ignored
    assert len(b["meshes"]) == 3 and [int(i[2]) for i in b["instances"]] == [0, 1, 2]
    v0, i0 = b["meshes"][0]
    assert len(v0) == 4 and list(i0) == [0, 1, 2, 0, 2, 3]                       # fan of the quad, vertices joined
    assert np.allclose(v0["uv"][2], [1, 0]) and np.allclose(v0["nrm"], [[0, 1, 0]] * 4)   # v flipped
    v1, i1 = b["meshes"][1]
    assert len(i1) == 3 + 6                                                       # a triangle + a fanned quad
    assert np.allclose(np.linalg.norm(v1["nrm"], axis=1), 1.0, atol=1e-6)
    assert np.linalg.det(b["instances"][0][0].reshape(4, 4).T[:3, :3]) < 0        # Y flip
    # unsupported extension / broken face index -> error codes
    (tmp_path / "bad.obj").write_text("v 0 0 0\nf 1 2 3\n")
    with pytest.raises(pt.B200ptError): pt.load_gltf(str(tmp_path / "bad.obj"))
    (tmp_path / "x.fbx").write_text("nope")
    with pytest.raises(pt.B200ptError): pt.load_gltf(str(tmp_path / "x.fbx"))


def test_decoders_and_importers_survive_corrupted_files(tmp_path):
    """Texture / scene files are untrusted input: flipped bytes, truncation and insertions must come back as error codes (or as a decoded
    image), never as a crash or an exception across the C-ABI.  (The same corpus generator was run under ASan / UBSan during development:
    it found an unchecked Huffman-table size and overflow in the IDCT of garbage coefficients, both fixed.)"""
    from PIL import Image
    rng = np.random.default_rng(123)
    img = (rng.random((29, 41, 3)) * 255).astype(np.uint8)
    Image.fromarray(img).save(tmp_path / "b.jpg", quality=80); Image.fromarray(img).save(tmp_path / "p.jpg", quality=80, progressive=True)
    Image.fromarray(img).save(tmp_path / "a.png"); util.write_rgbe(str(tmp_path / "e.hdr"), rng.random((7, 33, 3)).astype(np.float32) * 4)
    util.write_synthetic_gltf(tmp_path)
    (tmp_path / "o.obj").write_text("mtllib m.mtl\\nv 0 0 0\\nv 1 0 0\\nv 0 1 0\\nvt 0 0\\nvn 0 0 1\\nusemtl a\\nf 1/1/1 2/1/1 3/1/1\\n"); (tmp_path / "m.mtl").write_text("newmtl a\\nKd 1 0 0\\n")
    files = {"b.jpg": pt.decode_image, "p.jpg": pt.decode_image, "a.png": pt.decode_image, "e.hdr": pt.decode_hdr, "s.gltf": pt.load_gltf, "o.obj": pt.load_gltf}
    ok = bad = 0
    for it in range(480):
        name = list(files)[it % len(files)]; raw = bytearray((tmp_path / name).read_bytes())
        mode = int(rng.integers(0, 3))
        if mode == 0:
            for _ in range(int(rng.integers(1, 6))): raw[int(rng.integers(0, len(raw)))] = int(rng.integers(0, 256))
        elif mode == 1: raw = raw[:int(rng.integers(1, len(raw)))]
        else:
            a = int(rng.integers(0, len(raw))); raw[a:a] = bytes(rng.integers(0, 256, int(rng.integers(1, 9)), dtype=np.uint8))
        fn = tmp_path / ("mut" + os.path.splitext(name)[1]); fn.write_bytes(bytes(raw))
        try: files[name](str(fn)); ok += 1
        except pt.B200ptError: bad += 1
    assert ok + bad == 480 and bad > 100
