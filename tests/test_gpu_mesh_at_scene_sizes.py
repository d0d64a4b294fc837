"""The TSDF mesher (csrc/pm_mesh.cu: allocation, integration, extraction) at the scene sizes reconstruct --mesh meets, voxel
by voxel against the float64 oracle (oracle/mesh_oracle.py).

Rows.  Each builds an analytic scene (spheres, a room seen from inside, a ground disc): exact depth maps and a colour that
is a function of the world point, so no network runs.  Every row uses the voxel size reconstruct.default_mesh_voxel_size
picks for its depths, trunc 3 and min_weight 1, as the command does, and seeds the volume with back-projected depth pixels,
millions of them, as mesh_scan seeds it with the fused points.
  * dtu: 49 views on a DTU-like arc (fx 2892, depth about 600) of 1600x1200 around a sphere on a ground disc: two view
    chunks of the integration (32 + 17), blocks partly outside the images.
  * tnt: 100 views of 1920x1080 inside a spherical room: four chunks, camera planes cutting through allocated blocks.
  * eth3d: 24 views of a sphere, landscape 2688x1792 and portrait 1792x2688 alternating, each map in its own allocation and
    the views not listed in address order.
  * key-edge: four small spheres cut by the voxel range [-2^23, 2^23), 4 views of 640x480 each, so that blocks sit at block
    coordinate -2^20 and 2^20 - 1 on every axis and neighbour lookups cross the key range's edge (a key outside the range
    would alias a block on the other side).
  * big: a sphere of radius about 1200 voxels, 1920x1080 views enough to close it: over 2^24 vertices.

Checks per row.
  * Allocation: the keys equal mo.allocate.
  * Integration on sampled blocks, bit for bit (tsdf, weight, colour): a seeded random sample, the blocks whose corner
    projections lie within 2 pixels of an image border in some view, the blocks that straddle a camera plane (both at most
    SAMPLE_CAP, a seeded random choice beyond), and the blocks at the key range's edges.  Kernel and oracle perform the same
    float64 operations in the same order without fused multiply-adds, so any difference is a defect (a rounding tie in
    floor(u + 0.5) is evaluated identically on both sides).
  * Culling reach: a float64 mirror of block_may_see counts the (block, view) pairs culled by the image bounds, kept because
    the block straddles the camera plane (front < 8), and kept only by the one-pixel margin; each category a row is meant to
    reach is non-empty.
  * Extraction on the GPU's own volume against mo.marching_cubes_blocks: every block for the rows up to EXTRACT_ALL blocks,
    chunks at the start, middle and end of the key order for the big row, so compared faces carry indices above 2^24.
    Positions within 1e-6 relative, colours and faces exact.
  * The whole mesh twice, bit-identical; for the closed rows a closed oriented manifold, faces towards the cameras (all but
    slivers of under 1e-3 voxel faces in area, whose float32 corners carry no reliable orientation), radial error
    under RADIAL voxels; for the big row every face's edges at most sqrt(3) voxels long (plus the float32 rounding).

The CPU tests check that the checks reject planted errors and pin the rows' view counts, chunk counts and map sizes."""
import math
import time

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from patchmatchnet_b200 import ops, reconstruct
from tests import mesh_cases as mc

DEV = "cuda:0"
TRUNC = 3
VIEW_CHUNK = 32          # views the integration kernel stages per round
SAMPLE_RANDOM = 3000     # random blocks per row
SAMPLE_CAP = 4000        # border / straddle blocks per row at most
EXTRACT_ALL = 250000     # rows up to this many blocks are extracted and compared whole
EDGE_CHUNK = 3000        # blocks per compared chunk of the big row
LIMIT = 1 << 23          # voxel indices in [-2^23, 2^23)
# radial vertex error of the closed rows, in voxels.  Each view reads the depth of the pixel nearest to a voxel's projection,
# which moves its zero crossing along oblique rays; over millions of vertices the worst reaches 0.54 voxel on the eth3d row
# (0.45 on the small sphere of test_gpu_mesh, which keeps 0.5).  Exactness is the oracle comparisons' job.
RADIAL = 0.6


# ---- scenes -------------------------------------------------------------------------------------------------------------

def _look_at(centre, target, roll=0.0):
    E = mc.look_at(np.asarray(centre, np.float64), np.asarray(target, np.float64)).astype(np.float64)
    if roll == 0.0:
        return E.astype(np.float32)
    c, s = math.cos(roll), math.sin(roll)
    E[:2] = np.array([[c, -s], [s, c]]) @ E[:2]
    return E.astype(np.float32)


def _K(f, h, w):
    return np.array([[f, 0, w / 2 - 0.3], [0, f, h / 2 + 0.2], [0, 0, 1]], np.float32)


KEY_EDGE_ULP = 2.0 ** -11   # float32 spacing at the key-edge row's coordinates, about 8000 (2^23 voxels of 0.95e-3)


def _key_edge_group(centre, sign):
    """One sphere of the key-edge row (radius 0.014, about 14 voxels) and its 4 views along the axes, 0.3 away, from centres
    that differ from `centre` by multiples of KEY_EDGE_ULP."""
    Ks, Es, sizes = [], [], []
    q = lambda x: round(x / KEY_EDGE_ULP) * KEY_EDGE_ULP
    for k, lateral in ((0, 0.0), (1, 0.0), (2, 0.0), (0, q(0.005))):
        pos = centre.copy()
        pos[k] -= sign[k] * q(0.3)
        pos[(k + 1) % 3] -= sign[(k + 1) % 3] * lateral
        assert np.array_equal(pos.astype(np.float32).astype(np.float64), pos)
        Ks.append(_K(600.0, 480, 640)); Es.append(_look_at(pos, pos + np.eye(3)[k] * sign[k])); sizes.append((480, 640))
    return dict(Ks=Ks, Es=Es, sizes=sizes, prims=[("sphere", centre, 0.014)])


def _row_voxel_size(row):
    depths = [_render(row, v, "cpu")[0] for v in range(len(row["Ks"]))]
    return reconstruct.default_mesh_voxel_size(depths, row["Ks"])


def _row(name):
    """-> dict(Ks, Es, sizes [(H, W)], prims [(kind, ...)], stride, closed (centre, radius, +1 outward / -1 inward) or None,
    reach: culling categories the row must reach)."""
    rng = np.random.default_rng(7)
    Ks, Es, sizes = [], [], []
    if name == "dtu":
        centre = np.array([0.0, 0.0, 60.0])
        for el in np.radians(np.linspace(38, 68, 7)):
            for az in np.radians(np.linspace(-55, 55, 7)):
                pos = 600.0 * np.array([math.cos(el) * math.sin(az), -math.cos(el) * math.cos(az), math.sin(el)]) + centre * [1, 1, 0.5]
                Ks.append(_K(2892.0, 1200, 1600)); Es.append(_look_at(pos, centre * [1, 1, 0.5] + rng.normal(0, 8, 3)))
                sizes.append((1200, 1600))
        return dict(Ks=Ks, Es=Es, sizes=sizes, prims=[("sphere", centre, 60.0), ("disc", np.array([0.0, 0.0, 1.0]), np.zeros(3), 260.0)],
                    stride=4, closed=None, reach={"culled", "margin"})
    if name == "tnt":
        for d in mc.fibonacci(100):
            pos = rng.uniform(-0.5, 0.5, 3)
            Ks.append(_K(1165.0, 1080, 1920)); Es.append(_look_at(pos, pos + d, rng.uniform(-math.pi, math.pi))); sizes.append((1080, 1920))
        return dict(Ks=Ks, Es=Es, sizes=sizes, prims=[("sphere", np.zeros(3), 4.0)], stride=4, closed=(np.zeros(3), 4.0, -1),
                    reach={"culled", "straddle", "margin"})
    if name == "eth3d":
        centre = np.array([0.013, -0.021, 0.007])
        # close enough that no view meets the sphere at more than 60 degrees of incidence (nearest-pixel depths at grazing
        # incidence would move the surface by up to half a voxel)
        for v, d in enumerate(mc.fibonacci(24)):
            h, w = ((1792, 2688), (2688, 1792))[v % 2]
            Ks.append(_K(1000.0, h, w)); Es.append(_look_at(centre + 2.0 * d, centre, rng.uniform(-0.3, 0.3))); sizes.append((h, w))
        return dict(Ks=Ks, Es=Es, sizes=sizes, prims=[("sphere", centre, 1.0)], stride=4, closed=(centre, 1.0, 1), reach=set())
    if name == "key-edge":
        # cameras looking along the axes from exactly representable float32 centres, so E is exact in float32 and the maps,
        # hence the voxel size, do not depend on where the group sits: each sphere, of radius 14 voxels, is centred 2
        # voxels inside a corner of the voxel range for the voxel size the same group has at the origin
        s = _row_voxel_size(_key_edge_group(np.zeros(3), np.ones(3)))
        assert 2.0 ** (math.floor(math.log2((LIMIT - 3) * s)) - 23) == KEY_EDGE_ULP
        prims = []
        for sign in ((1, 1, 1), (-1, 1, 1), (1, -1, 1), (-1, -1, -1)):
            centre = np.float32(np.array(sign) * (LIMIT - 2) * s).astype(np.float64)
            g = _key_edge_group(centre, np.array(sign, np.float64))
            prims += g["prims"]; Ks += g["Ks"]; Es += g["Es"]; sizes += g["sizes"]
        return dict(Ks=Ks, Es=Es, sizes=sizes, prims=prims, stride=1, closed=None, reach={"culled"})
    if name == "big":
        for d in mc.fibonacci(150):
            Ks.append(_K(5000.0, 1080, 1920)); Es.append(_look_at(3.0 * d, np.zeros(3), rng.uniform(-math.pi, math.pi))); sizes.append((1080, 1920))
        return dict(Ks=Ks, Es=Es, sizes=sizes, prims=[("sphere", np.zeros(3), 1.0)], stride=6, closed=(np.zeros(3), 1.0, 1),
                    reach={"culled", "margin"})
    raise KeyError(name)


ROWS = ("dtu", "tnt", "eth3d", "key-edge", "big")


def _render(row, v, device):
    """-> (depth float32 [H,W], image float32 [3,H,W], world points float64 [H,W,3]) of view v: the nearest hit of the ray
    through each pixel centre, 0 where it hits nothing."""
    K = torch.tensor(row["Ks"][v], dtype=torch.float64, device=device)
    E = torch.tensor(row["Es"][v], dtype=torch.float64, device=device)
    H, W = row["sizes"][v]
    vv, uu = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=device), torch.arange(W, dtype=torch.float64, device=device),
                            indexing="ij")
    ray = torch.stack([uu, vv, torch.ones_like(uu)], -1) @ torch.linalg.inv(K).T  # camera frame, z = 1
    R, t = E[:3, :3], E[:3, 3]
    d = ray @ R                      # world direction (R^T ray)
    c = -(R.T @ t)                   # camera centre
    best = torch.full((H, W), math.inf, dtype=torch.float64, device=device)
    for p in row["prims"]:
        if p[0] == "sphere":
            C, r = torch.tensor(p[1], dtype=torch.float64, device=device), p[2]
            oc = c - C
            a, b, cc = (d * d).sum(-1), 2 * (d @ oc), oc @ oc - r * r
            disc = b * b - 4 * a * cc
            sq = torch.sqrt(disc.clamp(min=0))
            t1, t2 = (-b - sq) / (2 * a), (-b + sq) / (2 * a)
            hit = torch.where(t1 > 0, t1, torch.where(t2 > 0, t2, math.inf))
            hit = torch.where(disc >= 0, hit, math.inf)
        else:
            n, P0, rad = (torch.tensor(p[1], dtype=torch.float64, device=device), torch.tensor(p[2], dtype=torch.float64, device=device), p[3])
            hit = ((P0 - c) @ n) / (d @ n)
            X = c + hit[..., None] * d
            hit = torch.where((hit > 0) & ((X - P0).norm(dim=-1) <= rad), hit, math.inf)
        best = torch.minimum(best, hit)
    ok = torch.isfinite(best)
    depth = torch.where(ok, best, 0.0)
    X = c + depth[..., None] * d
    col = 0.5 + 0.4 * torch.stack([torch.sin(3 * X[..., 0]), torch.cos(2 * X[..., 1]), torch.sin(X[..., 2] + 1)])
    img = torch.where(ok, col, 0.0)
    return depth.float(), img.float(), torch.where(ok[..., None], X, math.nan)


def build_scene(name, device):
    """The row with its maps, voxel size and seeds on `device`: maps of the eth3d row each in its own allocation, listed in an
    order that is not their address order."""
    row = _row(name)
    V = len(row["Ks"])
    order = list(range(V))[::-1] if name == "eth3d" else list(range(V))
    depths, images, seeds = [None] * V, [None] * V, []
    for v in order:
        d, img, X = _render(row, v, device)
        depths[v], images[v] = d.clone(), img.clone()
        st = row["stride"]
        pts = X[::st, ::st].reshape(-1, 3)
        seeds.append(pts[torch.isfinite(pts[:, 0])].float())
    s = reconstruct.default_mesh_voxel_size(depths, row["Ks"])
    seeds = torch.cat(seeds)
    if name == "key-edge":  # the seeds whose truncation cube fits the voxel range, as the allocation requires
        p = seeds.double()
        seeds = seeds[((torch.floor((p - TRUNC * s) / s) >= -LIMIT) & (torch.floor((p + TRUNC * s) / s) < LIMIT)).all(1)]
    row.update(depths=depths, images=images, s=s, seeds=seeds.contiguous())
    return row


# ---- the culling mirror and the sample -----------------------------------------------------------------------------------

def cull_categories(keys, s, Ks, Es, sizes):
    """A float64 mirror of block_may_see (csrc/pm_mesh.cu) over every (block, view): -> dict of bool [n_blocks, V] tensors on
    keys' device: behind (no corner in front), straddle (kept: 0 < front < 8), culled (all in front, hull off the image by
    more than the margin), margin (kept, hull off the pixels [-0.5, W - 0.5) but within the one-pixel margin), near (all in
    front, a hull edge within 2 pixels of an image border line)."""
    dev = keys.device
    b = torch.from_numpy(mo.key_blocks(keys.cpu().numpy().view(np.uint64))).to(dev)
    lo, hi = (8 * b + 0.5) * s, (8 * b + 7.5) * s
    corners = torch.stack([torch.stack([(hi if c & 1 else lo)[:, 0], (hi if c & 2 else lo)[:, 1], (hi if c & 4 else lo)[:, 2]], -1)
                           for c in range(8)], 1)  # [B,8,3]
    out = {k: [] for k in ("behind", "straddle", "culled", "margin", "near")}
    for K, E, (H, W) in zip(Ks, Es, sizes):
        K = torch.tensor(np.asarray(K, np.float32), dtype=torch.float64, device=dev)
        Rt = torch.tensor(np.asarray(E, np.float32)[:3], dtype=torch.float64, device=dev)
        x, y, z = corners[..., 0], corners[..., 1], corners[..., 2]
        xc, yc, zc = (((Rt[i, 0] * x + Rt[i, 1] * y) + Rt[i, 2] * z) + Rt[i, 3] for i in range(3))
        front = zc > 0
        zs = torch.where(front, zc, 1.0)
        u = ((K[0, 0] * xc + K[0, 1] * yc) + K[0, 2] * zc) / zs
        w = ((K[1, 0] * xc + K[1, 1] * yc) + K[1, 2] * zc) / zs
        inf = torch.tensor(math.inf, dtype=torch.float64, device=dev)
        umin, umax = torch.where(front, u, inf).amin(1), torch.where(front, u, -inf).amax(1)
        vmin, vmax = torch.where(front, w, inf).amin(1), torch.where(front, w, -inf).amax(1)
        nf = front.sum(1)
        all8 = nf == 8
        culled = all8 & ((umax < -1.5) | (umin > W + 0.5) | (vmax < -1.5) | (vmin > H + 0.5))
        off = (umax < -0.5) | (umin >= W - 0.5) | (vmax < -0.5) | (vmin >= H - 0.5)
        near = all8 & (((umax + 0.5).abs() <= 2) | ((umin - (W - 0.5)).abs() <= 2) | ((vmax + 0.5).abs() <= 2) | ((vmin - (H - 0.5)).abs() <= 2))
        out["behind"].append(nf == 0); out["straddle"].append((nf > 0) & (nf < 8)); out["culled"].append(culled)
        out["margin"].append(all8 & ~culled & off); out["near"].append(near)
    return {k: torch.stack(v, 1) for k, v in out.items()}


def sample_blocks(cats, keys_np, rng):
    """Sorted block indices: SAMPLE_RANDOM random blocks, the near-border and the straddling blocks (each at most SAMPLE_CAP),
    and every block at the key range's edges.  -> (indices, counts of each part before the cap)."""
    n = len(keys_np)
    parts, counts = [rng.choice(n, min(n, SAMPLE_RANDOM), replace=False)], {}
    for cat in ("near", "straddle"):
        idx = torch.nonzero(cats[cat].any(1)).flatten().cpu().numpy()
        counts[cat] = len(idx)
        parts.append(rng.choice(idx, SAMPLE_CAP, replace=False) if len(idx) > SAMPLE_CAP else idx)
    b = mo.key_blocks(keys_np)
    edge = np.nonzero(((b == -mo.KEY_BIAS) | (b == mo.KEY_BIAS - 1)).any(1))[0]
    counts["edge"] = len(edge)
    parts.append(edge)
    return np.unique(np.concatenate(parts)), counts


# ---- checks ---------------------------------------------------------------------------------------------------------------

def check_volume(got, want):
    """got (tsdf, weight, colour [.,4]) and want (the oracle's tsdf, weight, colour [.,3]) as numpy: bit for bit."""
    tsdf, weight, colour = got
    wt, ww, wc = want
    bad = (tsdf.view(np.uint32) != wt.view(np.uint32)) | (weight != ww) | (colour[:, :3] != wc).any(1)
    assert not bad.any(), f"{bad.sum()} of {len(bad)} voxels differ, first at {np.nonzero(bad)[0][:8]}"
    assert (colour[:, 3] == 0).all()


def check_extraction(verts, faces, want):
    """GPU vertex records [nv,15] and faces [nf,3] (numpy) against mo.marching_cubes_blocks' output."""
    pos, col, wf, vid, fid = want
    assert len(vid) and len(fid)
    v = verts[vid]
    gp = v[:, :12].copy().view(np.float32)
    assert np.abs(gp - pos).max() <= 1e-6 * max(1.0, np.abs(pos).max())
    assert np.array_equal(v[:, 12:], col)
    assert np.array_equal(faces[fid], wf)


def check_closed_manifold_on_device(f, n_vertices):
    """mesh_cases.check_closed_manifold on the device, for meshes of millions of faces: faces int64 [nf,3]."""
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all()
    a = torch.cat([f[:, 0], f[:, 1], f[:, 2]])
    b = torch.cat([f[:, 1], f[:, 2], f[:, 0]])
    keys, _ = torch.sort(a * n_vertices + b)
    assert not (keys[1:] == keys[:-1]).any(), "a directed edge is used twice"
    rev = b * n_vertices + a
    pos = torch.searchsorted(keys, rev).clamp(max=len(keys) - 1)
    assert (keys[pos] == rev).all(), "an edge is not shared by two oppositely wound faces"
    assert torch.unique(f).numel() == n_vertices, "unreferenced vertices"
    assert n_vertices - len(keys) // 2 + len(f) == 2


# ---- CPU: the chunked oracle, the checks' sensitivity and the rows -------------------------------------------------------

@pytest.fixture(scope="module")
def sphere_volume():
    sc = mc.sphere_scene()
    s = 0.05
    keys = mo.allocate(sc["seeds"], s, TRUNC)
    return sc, s, keys, mo.integrate(keys, s, TRUNC, sc["depths"], sc["images"], sc["Ks"], sc["Es"])


@pytest.mark.parametrize("chunk", [1, 7, 64, 1000])
def test_chunked_oracle_equals_the_whole_volume_oracle(sphere_volume, chunk):
    sc, s, keys, vol = sphere_volume
    part = mo.integrate_blocks(keys[::-1], s, TRUNC, sc["depths"], sc["images"], sc["Ks"], sc["Es"], chunk=chunk)
    for a, b in zip(part, vol):  # any order of the blocks
        assert a.tobytes() == b.reshape(len(keys), 512, -1)[::-1].reshape(b.shape).tobytes()
    pos, col, faces = mo.marching_cubes(keys, s, *vol)
    got = mo.marching_cubes_blocks(keys, s, *vol, np.arange(len(keys)), chunk=chunk)
    assert got[0].tobytes() == pos.tobytes() and got[1].tobytes() == col.tobytes() and got[2].tobytes() == faces.tobytes()
    assert np.array_equal(got[3], np.arange(len(pos))) and np.array_equal(got[4], np.arange(len(faces)))
    for emit in (np.arange(0, len(keys), 5), np.array([len(keys) - 1]), np.arange(len(keys) // 3, len(keys) // 2)):
        p, c, f, vid, fid = mo.marching_cubes_blocks(keys, s, *vol, emit, chunk=chunk)
        assert p.tobytes() == pos[vid].tobytes() and c.tobytes() == col[vid].tobytes() and f.tobytes() == faces[fid].tobytes()


def test_oracles_do_not_alias_blocks_across_the_key_range_edge():
    """Blocks at x = 2^20 - 1 and at x = -2^20, y + 1: the neighbour key of the first at x = 2^20 would carry into y and name
    the second.  A surface cut by the edge meshes to the edge's last cube and no further, in both oracles."""
    e = mo.KEY_BIAS
    keys = np.sort(mo.block_key(np.array([[e - 1, 5, 9], [-e, 6, 9], [-e, 5, 9], [e - 1, 6, 9]])))
    G = len(keys) * 512
    c = mo.voxel_coords(keys)
    tsdf = np.where(c[:, 1] % 8 < 4, -0.5, 0.5).astype(np.float32)  # a plane y = const, cut by the edge
    vol = (tsdf, np.ones(G, np.float32), np.full((G, 3), 9, np.uint8))
    pos, col, faces = mo.marching_cubes(keys, 1.0, *vol)
    got = mo.marching_cubes_blocks(keys, 1.0, *vol, np.arange(len(keys)))
    assert got[2].tobytes() == faces.tobytes() and got[0].tobytes() == pos.tobytes()
    xs = pos[:, 0].astype(np.float64)
    assert xs.max() <= 8.0 * e - 0.5 and xs.min() >= -8.0 * e + 0.5 and len(faces) > 0


def test_checks_reject_planted_errors(sphere_volume):
    sc, s, keys, vol = sphere_volume
    got = (vol[0].copy(), vol[1].copy(), np.concatenate([vol[2], np.zeros((len(vol[2]), 1), np.uint8)], 1))
    check_volume(got, vol)
    i = int(np.nonzero(vol[1] > 0)[0][100])
    bad = (got[0], got[1].copy(), got[2])
    bad[1][i] += 1  # one voxel's weight off by one
    with pytest.raises(AssertionError):
        check_volume(bad, vol)
    # floor(u) in place of floor(u + 0.5): the principal point moved by half a pixel
    Kf = [k - np.array([[0, 0, 0.5], [0, 0, 0.5], [0, 0, 0]], np.float32) for k in sc["Ks"]]
    with pytest.raises(AssertionError):
        check_volume(got, mo.integrate(keys, s, TRUNC, sc["depths"], sc["images"], Kf, sc["Es"]))
    # one face index off by one
    ref = mo.marching_cubes_blocks(keys, s, *vol, np.arange(len(keys)))
    verts = np.concatenate([ref[0].view(np.uint8).reshape(-1, 12), ref[1]], 1)
    check_extraction(verts, ref[2], ref)
    f = ref[2].copy()
    f[len(f) // 2, 1] += 1
    with pytest.raises(AssertionError):
        check_extraction(verts, f, ref)


def test_integration_over_the_first_32_views_changes_the_dtu_sample():
    """A kernel that stopped after its first view chunk: the DTU row's random sample must see it."""
    sc = build_scene("dtu", "cpu")
    keys = mo.allocate(sc["seeds"].numpy()[::50], sc["s"], TRUNC)
    blocks = np.sort(np.random.default_rng(1).choice(len(keys), 300, replace=False))
    args = [[t.numpy() for t in sc["depths"]], [t.numpy() for t in sc["images"]], sc["Ks"], sc["Es"]]
    full = mo.integrate_blocks(keys[blocks], sc["s"], TRUNC, *args)
    first = mo.integrate_blocks(keys[blocks], sc["s"], TRUNC, *[a[:VIEW_CHUNK] for a in args])
    got = (first[0], first[1], np.concatenate([first[2], np.zeros((len(first[2]), 1), np.uint8)], 1))
    with pytest.raises(AssertionError):
        check_volume(got, full)
    assert (full[1] > VIEW_CHUNK).any()


# (views, view chunks of the integration, map sizes (H, W))
ROW_TABLE = {"dtu": (49, 2, {(1200, 1600)}), "tnt": (100, 4, {(1080, 1920)}), "eth3d": (24, 1, {(1792, 2688), (2688, 1792)}),
             "key-edge": (16, 1, {(480, 640)}), "big": (150, 5, {(1080, 1920)})}


@pytest.mark.parametrize("name", ROWS)
def test_row_table(name):
    row = _row(name)
    V = len(row["Ks"])
    views, chunks, sizes = ROW_TABLE[name]
    assert (V, -(-V // VIEW_CHUNK), set(row["sizes"])) == (views, chunks, sizes)
    assert len(row["Es"]) == V and all(k.shape == (3, 3) and e.shape == (4, 4) for k, e in zip(row["Ks"], row["Es"]))
    if name == "eth3d":
        assert row["sizes"][0] != row["sizes"][1]


# ---- GPU ------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module", params=ROWS)
def scene(request):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    sc = build_scene(request.param, DEV)
    sc["name"] = request.param
    sc["keys"] = ops.tsdf_allocate(sc["seeds"], sc["s"], TRUNC)
    yield sc
    print(f"[{request.param}] {time.perf_counter() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB")
    sc.clear()
    torch.cuda.empty_cache()


def _np_keys(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.mark.gpu
def test_allocation_and_sampled_integration(scene):
    sc = scene
    keys = _np_keys(sc["keys"])
    assert np.array_equal(keys, mo.allocate(sc["seeds"].cpu().numpy(), sc["s"], TRUNC))
    if sc["name"] == "eth3d":
        ptrs = [d.data_ptr() for d in sc["depths"]]
        assert ptrs != sorted(ptrs)
    vol = ops.tsdf_integrate(sc["keys"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], sc["s"], TRUNC)
    cats = cull_categories(sc["keys"], sc["s"], sc["Ks"], sc["Es"], sc["sizes"])
    reach = {k: int(v.sum()) for k, v in cats.items()}
    blocks, counts = sample_blocks(cats, keys, np.random.default_rng(3))
    print(f"[{sc['name']}] s {sc['s']:.6g}, {len(sc['seeds'])} seeds, {len(keys)} blocks; (block, view) pairs {reach}; "
          f"sampled {len(blocks)} blocks (before the cap: {counts})")
    for cat in sc["reach"]:
        assert reach[cat] > 0, cat
    if sc["name"] == "key-edge":
        b = mo.key_blocks(keys)
        for a in range(3):
            assert (b[:, a] == -mo.KEY_BIAS).any() and (b[:, a] == mo.KEY_BIAS - 1).any()
    idx = torch.from_numpy(blocks).to(DEV)
    got = tuple(t.view(len(keys), 512, -1)[idx].reshape((len(blocks) * 512,) + t.shape[1:]).cpu().numpy() for t in vol)
    want = mo.integrate_blocks(keys[blocks], sc["s"], TRUNC, [d.cpu().numpy() for d in sc["depths"]],
                               [i.cpu().numpy() for i in sc["images"]], sc["Ks"], sc["Es"])
    check_volume(got, want)
    assert (want[1] > 0).mean() > 0.2
    sc["vol"] = vol


@pytest.mark.gpu
def test_extraction_on_the_gpu_volume(scene):
    sc = scene
    if "vol" not in sc:
        sc["vol"] = ops.tsdf_integrate(sc["keys"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], sc["s"], TRUNC)
    verts, faces = ops.tsdf_extract(sc["keys"], *sc["vol"], sc["s"], 1)
    keys = _np_keys(sc["keys"])
    n = len(keys)
    if n <= EXTRACT_ALL:
        emit = np.arange(n)
    else:
        emit = np.concatenate([np.arange(EDGE_CHUNK), np.arange(n // 2, n // 2 + EDGE_CHUNK), np.arange(n - EDGE_CHUNK, n)])
    want = mo.marching_cubes_blocks(keys, sc["s"], *(t.cpu().numpy() for t in sc["vol"]), emit)
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    if n <= EXTRACT_ALL:
        assert len(want[3]) == len(v) and len(want[4]) == len(f)
    else:
        assert f[want[4]].max() >= 1 << 24 and len(v) > 1 << 24
    check_extraction(v, f, want)
    print(f"[{sc['name']}] {n} blocks, {len(v)} vertices, {len(f)} faces; compared {len(emit)} blocks: {len(want[3])} vertices, "
          f"{len(want[4])} faces")
    sc.pop("vol")
    sc["mesh"] = (verts, faces)


@pytest.mark.gpu
def test_whole_mesh(scene):
    sc = scene
    a = ops.tsdf_mesh(sc["seeds"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], sc["s"], TRUNC, 1)
    if "mesh" in sc:  # integration and extraction called one by one give the same mesh
        assert torch.equal(a[0], sc["mesh"][0]) and torch.equal(a[1], sc["mesh"][1])
        sc.pop("mesh")
    b = ops.tsdf_mesh(sc["seeds"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], sc["s"], TRUNC, 1)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    del b
    s = sc["s"]
    pos = a[0][:, :12].contiguous().view(torch.float32).double()
    f = a[1].long()
    if sc["closed"] is None:
        return
    check_closed_manifold_on_device(f, len(pos))
    centre, radius, sign = sc["closed"]
    cen = torch.tensor(centre, dtype=torch.float64, device=DEV)
    p = pos[f]
    n = torch.linalg.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    # faces towards the cameras; a sliver whose float32 corners nearly coincide has no reliable orientation
    solid = n.norm(dim=1) >= 1e-3 * s * s
    assert (sign * (n * (p.mean(1) - cen)).sum(1) > 0)[solid].all()
    del p, n
    radial = (pos - cen).norm(dim=1) - radius
    assert radial.abs().max() < RADIAL * s, float(radial.abs().max() / s)
    if sc["name"] == "big":  # a corrupted vertex index makes a long edge
        edges = torch.cat([(pos[f[:, i]] - pos[f[:, (i + 1) % 3]]).norm(dim=1) for i in range(3)])
        assert edges.max() <= math.sqrt(3) * s + 2 * 2.0 ** -23 * float(pos.abs().max()), float(edges.max() / s)
