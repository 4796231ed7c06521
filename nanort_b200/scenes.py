"""Deterministic synthetic scenes, cameras and ray sets for BASELINE.json's configs.

The reference ships no benchmark scenes besides two OBJ files, so the workloads
of BASELINE.json ("Cornell box (~32 tris)", "100K-triangle sphere-grid",
"1M-triangle procedural terrain", "10M-triangle instanced scene") are generated
here (SURVEY.md section 8d).  Camera rays follow the pinhole construction of
the reference path tracer (examples/path_tracer/main.cc:809-817, 839-849), AO
rays its hit-point / normal / cosine-hemisphere pieces (main.cc:860, 306-312,
878-881, 216-250, 675-701), with a counter-based hash instead of libc rand().

Everything is float32 / uint32 and laid out exactly as nanort consumes it:
vertices [nv,3] float32 (stride 12), faces [nf,3] uint32, rays as 36-byte
nanort::Ray records (structured dtype RAY_DTYPE), hits as 16-byte
nanort::TriangleIntersection records (HIT_DTYPE).
"""
from __future__ import annotations

import numpy as np

RAY_DTYPE = np.dtype(
    [("org", "<f4", (3,)), ("dir", "<f4", (3,)), ("min_t", "<f4"), ("max_t", "<f4"), ("type", "<u4")]
)
HIT_DTYPE = np.dtype([("u", "<f4"), ("v", "<f4"), ("t", "<f4"), ("prim_id", "<u4")])
NODE_DTYPE = np.dtype(
    [("bmin", "<f4", (3,)), ("bmax", "<f4", (3,)), ("flag", "<i4"), ("axis", "<i4"), ("data", "<u4", (2,))]
)
assert RAY_DTYPE.itemsize == 36 and HIT_DTYPE.itemsize == 16 and NODE_DTYPE.itemsize == 40


# ----------------------------------------------------------------------------- hashing
def hash_u32(x: np.ndarray) -> np.ndarray:
    """lowbias32 integer hash, vectorised (same function as csrc/render.cu:hash_u32)."""
    x = np.asarray(x, dtype=np.uint64) & 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x846CA68B) & 0xFFFFFFFF
    x ^= x >> 16
    return x.astype(np.uint32)


def rand01(index: np.ndarray, dim: int, seed: int) -> np.ndarray:
    """Uniform float32 in [0,1) from (index, dim, seed); 24 random bits."""
    idx = np.asarray(index, dtype=np.uint64)
    k = (idx * 0x9E3779B1 + np.uint64(dim) * 0x85EBCA77 + np.uint64(seed) * 0xC2B2AE3D) & 0xFFFFFFFF
    h = hash_u32(hash_u32(k) ^ np.uint32(0x27D4EB2F))
    return ((h >> 8).astype(np.float32)) * np.float32(1.0 / 16777216.0)


def rand_ps(pix: np.ndarray, smp: np.ndarray, dim: int, seed: int) -> np.ndarray:
    """Uniform float32 in [0,1) keyed by (pixel, sample, dimension, seed); all arithmetic wraps at 32 bits.
    Same function as csrc/render.cu:rand_ps."""
    M = 0xFFFFFFFF
    pix = np.asarray(pix, dtype=np.uint64) & M
    smp = np.asarray(smp, dtype=np.uint64) & M
    h = hash_u32((pix + ((seed * 0x9E3779B1) & M)) & M).astype(np.uint64)
    h = hash_u32((h + ((smp * 0x85EBCA77) & M) + ((dim * 0xC2B2AE3D) & M)) & M)
    return ((h >> 8).astype(np.float32)) * np.float32(1.0 / 16777216.0)


# ----------------------------------------------------------------------------- meshes
def _quad(v, f, a, b, c, d):
    base = len(v)
    v.extend([a, b, c, d])
    f.append((base, base + 1, base + 2))
    f.append((base, base + 2, base + 3))


def _box(v, f, lo, hi, yaw=0.0):
    lo = np.asarray(lo, np.float64)
    hi = np.asarray(hi, np.float64)
    cx, cz = 0.5 * (lo[0] + hi[0]), 0.5 * (lo[2] + hi[2])
    cs, sn = np.cos(yaw), np.sin(yaw)

    def P(x, y, z):
        dx, dz = x - cx, z - cz
        return (cx + cs * dx - sn * dz, y, cz + sn * dx + cs * dz)

    x0, y0, z0 = lo
    x1, y1, z1 = hi
    _quad(v, f, P(x0, y0, z1), P(x1, y0, z1), P(x1, y1, z1), P(x0, y1, z1))  # front
    _quad(v, f, P(x1, y0, z0), P(x0, y0, z0), P(x0, y1, z0), P(x1, y1, z0))  # back
    _quad(v, f, P(x0, y0, z0), P(x0, y0, z1), P(x0, y1, z1), P(x0, y1, z0))  # left
    _quad(v, f, P(x1, y0, z1), P(x1, y0, z0), P(x1, y1, z0), P(x1, y1, z1))  # right
    _quad(v, f, P(x0, y1, z1), P(x1, y1, z1), P(x1, y1, z0), P(x0, y1, z0))  # top
    _quad(v, f, P(x0, y0, z0), P(x1, y0, z0), P(x1, y0, z1), P(x0, y0, z1))  # bottom


def cornell():
    """Config 1: 5 walls + 2 boxes = 34 triangles inside [-5,5]x[0,10]x[-5,5]."""
    v, f = [], []
    _quad(v, f, (-5, 0, 5), (5, 0, 5), (5, 0, -5), (-5, 0, -5))  # floor
    _quad(v, f, (-5, 10, -5), (5, 10, -5), (5, 10, 5), (-5, 10, 5))  # ceiling
    _quad(v, f, (-5, 0, -5), (5, 0, -5), (5, 10, -5), (-5, 10, -5))  # back
    _quad(v, f, (-5, 0, 5), (-5, 0, -5), (-5, 10, -5), (-5, 10, 5))  # left
    _quad(v, f, (5, 0, -5), (5, 0, 5), (5, 10, 5), (5, 10, -5))  # right
    _box(v, f, (-3.4, 0.0, -3.2), (-0.6, 6.0, -0.4), yaw=0.3)  # tall box
    _box(v, f, (0.7, 0.0, 0.3), (3.5, 2.8, 3.1), yaw=-0.3)  # short box
    return np.asarray(v, np.float32), np.asarray(f, np.uint32)


def uv_sphere(n_lon=25, n_lat=21, radius=0.4):
    """2*n_lon*(n_lat-1) triangles (1000 for the defaults)."""
    verts = [(0.0, radius, 0.0)]
    for j in range(1, n_lat):
        th = np.pi * j / n_lat
        for i in range(n_lon):
            ph = 2.0 * np.pi * i / n_lon
            verts.append((radius * np.sin(th) * np.cos(ph), radius * np.cos(th), radius * np.sin(th) * np.sin(ph)))
    verts.append((0.0, -radius, 0.0))
    south = len(verts) - 1
    faces = []

    def ring(j, i):
        return 1 + (j - 1) * n_lon + (i % n_lon)

    for i in range(n_lon):
        faces.append((0, ring(1, i + 1), ring(1, i)))
    for j in range(1, n_lat - 1):
        for i in range(n_lon):
            a, b, c, d = ring(j, i), ring(j, i + 1), ring(j + 1, i + 1), ring(j + 1, i)
            faces.append((a, b, c))
            faces.append((a, c, d))
    for i in range(n_lon):
        faces.append((south, ring(n_lat - 1, i), ring(n_lat - 1, i + 1)))
    return np.asarray(verts, np.float64), np.asarray(faces, np.int64)


def sphere_grid(nx=10, nz=10, n_lon=25, n_lat=21, radius=0.4, floor=True, offset=(0.0, 0.0, 0.0)):
    """Config 2: nx*nz UV spheres of 1000 triangles on a unit lattice + a 2-triangle floor
    (100,002 triangles for the defaults)."""
    sv, sf = uv_sphere(n_lon, n_lat, radius)
    nv = len(sv)
    vs, fs = [], []
    k = 0
    for iz in range(nz):
        for ix in range(nx):
            c = np.array([ix - 0.5 * (nx - 1), radius, iz - 0.5 * (nz - 1)])
            vs.append(sv + c)
            fs.append(sf + k * nv)
            k += 1
    if floor:
        hx, hz = 0.5 * nx + 0.5, 0.5 * nz + 0.5
        base = k * nv
        vs.append(np.array([(-hx, 0, hz), (hx, 0, hz), (hx, 0, -hz), (-hx, 0, -hz)], np.float64))
        fs.append(np.array([(base, base + 1, base + 2), (base, base + 2, base + 3)], np.int64))
    v = np.concatenate(vs) + np.asarray(offset, np.float64)
    return v.astype(np.float32), np.concatenate(fs).astype(np.uint32)


def _value_noise(n, cells, seed):
    """Bilinear value noise on an (n+1)x(n+1) grid with `cells` lattice cells per side."""
    g = np.arange(n + 1, dtype=np.float64) * (cells / n)
    i0 = np.minimum(np.floor(g).astype(np.int64), cells - 1)
    fr = g - i0
    fr = fr * fr * (3.0 - 2.0 * fr)
    lat_idx = np.arange((cells + 1) * (cells + 1), dtype=np.uint64)
    lat = rand01(lat_idx, 0, seed).astype(np.float64).reshape(cells + 1, cells + 1)
    a = lat[np.ix_(i0, i0)]
    b = lat[np.ix_(i0, i0 + 1)]
    c = lat[np.ix_(i0 + 1, i0)]
    d = lat[np.ix_(i0 + 1, i0 + 1)]
    fx = fr[None, :]
    fz = fr[:, None]
    return (a * (1 - fx) + b * fx) * (1 - fz) + (c * (1 - fx) + d * fx) * fz


def terrain(n=708, size=10.0, height=1.2, seed=7):
    """Config 3: n x n heightfield quads -> 2*n*n triangles (708 -> 1,002,528); fBm heights."""
    h = np.zeros((n + 1, n + 1), np.float64)
    amp, cells = 1.0, 4
    for octave in range(6):
        h += amp * _value_noise(n, cells, seed + octave)
        amp *= 0.5
        cells *= 2
    h = (h - h.min()) / (h.max() - h.min()) * height
    xs = (np.arange(n + 1, dtype=np.float64) / n - 0.5) * size
    X, Z = np.meshgrid(xs, xs)
    v = np.stack([X, h, Z], axis=-1).reshape(-1, 3)
    iz, ix = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a = (iz * (n + 1) + ix).reshape(-1)
    b = a + 1
    c = a + (n + 1) + 1
    d = a + (n + 1)
    f = np.empty((2 * n * n, 3), np.int64)
    f[0::2] = np.stack([a, c, b], axis=1)
    f[1::2] = np.stack([a, d, c], axis=1)
    return v.astype(np.float32), f.astype(np.uint32)


def instanced(copies_x=10, copies_z=10):
    """Config 4: copies_x*copies_z translated copies of the config-2 sphere grid FLATTENED into one
    soup (10,000,200 triangles for 10x10) -- nanort's core has no instancing (SURVEY.md 8d)."""
    v0, f0 = sphere_grid()
    nv = len(v0)
    vs, fs = [], []
    k = 0
    for iz in range(copies_z):
        for ix in range(copies_x):
            off = np.array([(ix - 0.5 * (copies_x - 1)) * 11.0, 0.0, (iz - 0.5 * (copies_z - 1)) * 11.0], np.float32)
            vs.append(v0 + off)
            fs.append(f0 + np.uint32(k * nv))
            k += 1
    return np.concatenate(vs).astype(np.float32), np.concatenate(fs).astype(np.uint32)


def xform(translate=(0, 0, 0), scale=(1, 1, 1), yaw=0.0, pitch=0.0):
    """4x4 float32 in the reference scene graph's convention (examples/nanosg/nanosg.h:214-222): row-vector
    form, p' = p . M, translation in row 3."""
    cy, sy, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    ry = np.array([[cy, 0, -sy], [0, 1, 0], [sy, 0, cy]])
    rx = np.array([[1, 0, 0], [0, cp, sp], [0, -sp, cp]])
    m = np.eye(4)
    m[:3, :3] = np.diag(scale) @ rx @ ry
    m[3, :3] = translate
    return m.astype(np.float32)


def instances_grid(copies_x=10, copies_z=10, base=None):
    """Config 4 as a two-level scene: copies_x*copies_z translated instances of ONE config-2 sphere grid
    (the same placement `instanced()` flattens)."""
    v0, f0 = base if base is not None else sphere_grid()
    out = []
    for iz in range(copies_z):
        for ix in range(copies_x):
            off = ((ix - 0.5 * (copies_x - 1)) * 11.0, 0.0, (iz - 0.5 * (copies_z - 1)) * 11.0)
            out.append((v0, f0, xform(translate=off)))
    return out


def instances_mixed(n=24, seed=11, tris_per_sphere=(9, 7)):
    """Small two-level parity scene: n instances over three base meshes (two spheres of different
    tessellation and the Cornell box) with translation, non-uniform scale and rotation; boxes overlap."""
    a = uv_sphere(*tris_per_sphere, radius=1.0)
    b = uv_sphere(13, 11, radius=0.7)
    c = cornell()
    bases = [a, b, (c[0] * np.float32(0.2), c[1])]
    i = np.arange(n, dtype=np.int64)
    r = [rand01(i, k, seed) for k in range(9)]
    out = []
    for k in range(n):
        v, f = bases[k % 3]
        t = ((r[0][k] - 0.5) * 12.0, (r[1][k] - 0.5) * 4.0, (r[2][k] - 0.5) * 12.0)
        sc = (0.5 + 1.5 * r[3][k], 0.5 + 1.5 * r[4][k], 0.5 + 1.5 * r[5][k])
        out.append((v, f, xform(t, sc, yaw=float(r[6][k]) * 6.2831853, pitch=(float(r[7][k]) - 0.5) * 1.5)))
    return out


def instances_row(n=80):
    """n unit-ish spheres in a row along x plus exact duplicates: a ray down the row pierces more than the 64
    boxes the reference keeps (nanosg.h:787) and meets exact box-entry ties."""
    v, f = uv_sphere(9, 7, radius=0.45)
    out = [(v, f, xform(translate=(float(k), 0.0, 0.0))) for k in range(n)]
    out += [(v, f, xform(translate=(float(k), 0.0, 0.0))) for k in (3, 3, 10, 40)]  # coincident instances
    return out


def with_area_light(verts, faces, center, half_x, half_z):
    """Appends a downward-facing emissive quad (2 triangles, the LAST two faces) -- the mesh light the
    reference path tracer samples (examples/path_tracer/main.cc:323-392).  Returns (verts, faces,
    light_first_face, light_n_faces)."""
    cx, cy, cz = center
    q = np.array([(cx - half_x, cy, cz - half_z), (cx + half_x, cy, cz - half_z), (cx + half_x, cy, cz + half_z),
                  (cx - half_x, cy, cz + half_z)], np.float32)
    base = len(verts)
    lf = np.array([(base, base + 1, base + 2), (base, base + 2, base + 3)], np.uint32)  # normal (0,-1,0)
    return (np.concatenate([verts, q]).astype(np.float32), np.concatenate([faces, lf]).astype(np.uint32),
            len(faces), 2)


MATERIAL_DTYPE = np.dtype([("diffuse", "<f4", (3,)), ("specular", "<f4", (3,)), ("transmittance", "<f4", (3,)),
                           ("emission", "<f4", (3,)), ("ior", "<f4"), ("dissolve", "<f4"), ("pad", "<f4", (2,))])
assert MATERIAL_DTYPE.itemsize == 64


def material(diffuse=(0, 0, 0), specular=(0, 0, 0), transmittance=(0, 0, 0), emission=(0, 0, 0), ior=1.0, dissolve=0.0):
    """One tinyobj-style material record as the reference path tracer reads it (main.cc:884-892).  NOTE the
    reference's convention: dissolve weighs the REFRACTION lobe, (1 - dissolve) the diffuse one (main.cc:908-913),
    exactly like examples/common/cornellbox_suzanne_lucy.mtl uses it (d 0 = diffuse, d 1 = glass)."""
    m = np.zeros(1, MATERIAL_DTYPE)
    m["diffuse"], m["specular"], m["transmittance"], m["emission"] = diffuse, specular, transmittance, emission
    m["ior"], m["dissolve"] = ior, dissolve
    return m


def cornell_with_materials():
    """The 34-triangle Cornell box + a ceiling light, with the material set of the reference's
    cornellbox_suzanne_lucy.mtl: grey floor/ceiling/back, red and green walls, a mirror-like tall box, a glass
    short box, an emitter.  Returns (verts, faces, materials, material_ids, emissive_faces)."""
    v, f = cornell()
    v, f, l0, ln = with_area_light(v, f, (0.0, 9.99, 0.0), 1.5, 1.5)
    mats = np.concatenate([
        material(diffuse=(0.8, 0.8, 0.8)),                                    # 0 grey
        material(diffuse=(0.8, 0.05, 0.05)),                                  # 1 red
        material(diffuse=(0.023, 0.41, 0.048)),                               # 2 green
        material(specular=(1.0, 1.0, 1.0)),                                   # 3 "Monkey": pure specular
        material(specular=(0.9, 0.9, 1.0), transmittance=(0.9, 0.9, 1.0), ior=1.5, dissolve=1.0),  # 4 "Reflective" glass
        material(emission=(15.0, 15.0, 15.0)),                                # 5 light
        material(diffuse=(1.0, 0.8, 0.8), specular=(0.2, 0.2, 0.2)),          # 6 "Lucy"
    ])
    ids = np.zeros(len(f), np.uint32)
    ids[0:2] = 6      # floor: diffuse + a little specular
    ids[2:6] = 0      # ceiling, back
    ids[6:8] = 1      # left wall
    ids[8:10] = 2     # right wall
    ids[10:22] = 3    # tall box
    ids[22:34] = 4    # short box
    ids[l0:l0 + ln] = 5
    emissive = np.nonzero(mats["emission"][ids].sum(axis=1) > 0)[0].astype(np.uint32)
    return v, f, mats, ids, emissive


# ----------------------------------------------------------------------------- cameras
def _normalize(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def look_at(org, target, up=(0, 1, 0), fov_y_deg=45.0, aspect=1.0):
    """Returns the 12-float camera block {org, right*sx, up*sy, forward} used by both the numpy
    generator below and csrc/render.cu:gen_primary."""
    fwd = _normalize(np.asarray(target, np.float64) - np.asarray(org, np.float64))
    right = _normalize(np.cross(fwd, np.asarray(up, np.float64)))
    upv = np.cross(right, fwd)
    sy = 2.0 * np.tan(np.radians(fov_y_deg) * 0.5)
    sx = sy * aspect
    return np.concatenate([np.asarray(org, np.float64), right * sx, upv * sy, fwd]).astype(np.float32)


def scene_camera(name: str, width: int, height: int) -> np.ndarray:
    aspect = width / float(height)
    if name == "cornell":
        # examples/path_tracer/main.cc:809-817: org (0,5,20), dir = normalize(px/W-.5, py/H-.5, -1)
        return np.array([0, 5, 20, 1, 0, 0, 0, 1, 0, 0, 0, -1], np.float32)
    if name == "sphere_grid":
        return look_at((0.0, 6.5, 11.0), (0.0, 0.2, 0.0), fov_y_deg=40.0, aspect=aspect)
    if name == "terrain":
        return look_at((0.0, 4.0, 8.5), (0.0, 0.3, 0.0), fov_y_deg=42.0, aspect=aspect)
    if name == "instanced":
        return look_at((0.0, 60.0, 95.0), (0.0, 0.0, 0.0), fov_y_deg=42.0, aspect=aspect)
    raise KeyError(name)


SCENES = {
    "cornell": cornell,
    "sphere_grid": sphere_grid,
    "terrain": terrain,
    "instanced": instanced,
}


def make_scene(name: str, **kw):
    v, f = SCENES[name](**kw)
    return np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.uint32)


# ----------------------------------------------------------------------------- UV atlases (texel cast / bake)
# A UV mesh in the layout of the reference's uv_raster (SetupVerticesForUVRaster, examples/uv_raster/main.cc:236-254):
# vertex 3i + k = (u, v, 0) of corner k of face i, face i = (3i, 3i+1, 3i+2).
def _uv_mesh(uv):
    uv = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    verts = np.zeros((uv.shape[0] * 3, 3), np.float32)
    verts[:, :2] = uv.reshape(-1, 2)
    return verts, np.arange(uv.shape[0] * 3, dtype=np.uint32).reshape(-1, 3)


def planar_uv(verts, faces):
    """Face-varying UVs of a heightfield such as terrain(): each corner's (x, z) normalised to [0, 1].  Returns the UV
    mesh (verts [3n, 3], faces [n, 3])."""
    v = np.asarray(verts, np.float64)
    lo, hi = v.min(axis=0), v.max(axis=0)
    xz = (v[:, [0, 2]] - lo[[0, 2]]) / np.maximum(hi[[0, 2]] - lo[[0, 2]], 1e-30)
    return _uv_mesh(xz[np.asarray(faces)])


def per_face_atlas(n_faces, gutter=0.15):
    """One right-triangle chart per face for meshes without UVs: faces fill a cols x cols grid of cells (cols =
    ceil(sqrt(n_faces))), row-major from (0, 0); face i covers the lower-left half of its cell, inset by `gutter`
    times the cell size, so that no two charts touch.  Returns the UV mesh (verts [3n, 3], faces [n, 3])."""
    cols = max(1, int(np.ceil(np.sqrt(n_faces))))
    cell = 1.0 / cols
    i = np.arange(n_faces)
    x0 = (i % cols) * cell + gutter * cell
    y0 = (i // cols) * cell + gutter * cell
    e = cell * (1.0 - 2.0 * gutter)
    uv = np.stack([np.stack([x0, y0], 1), np.stack([x0 + e, y0], 1), np.stack([x0, y0 + e], 1)], axis=1)
    return _uv_mesh(uv)


# ----------------------------------------------------------------------------- rays
def primary_rays(cam, width, height, spp=1, seed=1, pixels=None, sample0=0, min_t=1e-3, max_t=1e30):
    """Jittered pinhole rays, ray index = (pixel * spp + s).  `pixels` optionally restricts to a
    flat array of pixel indices (y*width+x)."""
    cam = np.asarray(cam, np.float32)
    if pixels is None:
        pixels = np.arange(width * height, dtype=np.int64)
    pixels = np.asarray(pixels, np.int64)
    pix = np.repeat(pixels, spp)
    smp = np.tile(np.arange(sample0, sample0 + spp, dtype=np.int64), len(pixels))
    jx = rand_ps(pix, smp, 0, seed)
    jy = rand_ps(pix, smp, 1, seed)
    px = (pix % width).astype(np.float32)
    py = (pix // width).astype(np.float32)
    sx = (px + jx) / np.float32(width) - np.float32(0.5)
    sy = np.float32(0.5) - (py + jy) / np.float32(height)
    d = cam[3:6][None, :] * sx[:, None] + cam[6:9][None, :] * sy[:, None] + cam[9:12][None, :]
    d = d.astype(np.float32)
    # the device's arithmetic (CameraRays in csrc/wavefront.cuh, gen_camera_kernel in csrc/path.cu): one reciprocal,
    # three multiplies -- a division per component differs from it in the last bit for about a third of the rays
    inv = (np.float32(1.0) / np.sqrt(((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float32))).astype(np.float32)
    d = (d * inv[:, None]).astype(np.float32)
    rays = np.zeros(len(pix), RAY_DTYPE)
    rays["org"] = cam[0:3]
    rays["dir"] = d
    rays["min_t"] = np.float32(min_t)
    rays["max_t"] = np.float32(max_t)
    rays["type"] = 1
    return rays


def ao_rays(verts, faces, rays, hits, mask, seed=2, min_t=1e-3, max_t=1.0):
    """One cosine-hemisphere AO ray per hit (closest-hit query with max_t = AO radius, exactly how
    CheckForOccluder works, examples/path_tracer/main.cc:675-701).  Returns (ao_rays, src_index)."""
    idx = np.nonzero(mask)[0]
    r = rays[idx]
    h = hits[idx]
    o = r["org"].astype(np.float32)
    d = r["dir"].astype(np.float32)
    P = o + d * h["t"][:, None]
    f = faces[h["prim_id"]]
    p0, p1, p2 = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    n = np.cross(p1 - p0, p2 - p0).astype(np.float32)
    ln = np.sqrt((n * n).sum(axis=1))
    ln[ln == 0] = 1.0
    n = n / ln[:, None]
    flip = (n * d).sum(axis=1) > 0
    n[flip] = -n[flip]
    # orthonormal basis (Frisvad-style, cf. revisedONB main.cc:216-236)
    sgn = np.where(n[:, 2] >= 0, 1.0, -1.0).astype(np.float32)
    a = -1.0 / (sgn + n[:, 2])
    b = n[:, 0] * n[:, 1] * a
    t1 = np.stack([1.0 + sgn * n[:, 0] * n[:, 0] * a, sgn * b, -sgn * n[:, 0]], axis=1).astype(np.float32)
    t2 = np.stack([b, sgn + n[:, 1] * n[:, 1] * a, -n[:, 1]], axis=1).astype(np.float32)
    u1 = rand01(idx, 2, seed)
    u2 = rand01(idx, 3, seed)
    rr = np.sqrt(u1)
    ph = np.float32(2.0 * np.pi) * u2
    lx, ly, lz = rr * np.cos(ph), rr * np.sin(ph), np.sqrt(np.maximum(0.0, 1.0 - u1))
    w = (t1 * lx[:, None] + t2 * ly[:, None] + n * lz[:, None]).astype(np.float32)
    w /= np.sqrt((w * w).sum(axis=1))[:, None]
    out = np.zeros(len(idx), RAY_DTYPE)
    out["org"] = P.astype(np.float32)
    out["dir"] = w.astype(np.float32)
    out["min_t"] = np.float32(min_t)
    out["max_t"] = np.float32(max_t)
    out["type"] = 2
    return out, idx


def incoherent_rays(bmin, bmax, n, seed=3, axis_parallel_fraction=1.0 / 32):
    """Random interior rays incl. axis-parallel and -0.0 direction components and finite max_t
    (the ray family of SURVEY.md probe P11)."""
    bmin = np.asarray(bmin, np.float32)
    bmax = np.asarray(bmax, np.float32)
    i = np.arange(n, dtype=np.int64)
    o = np.stack([rand01(i, k, seed) for k in range(3)], axis=1) * (bmax - bmin) + bmin
    z = rand01(i, 3, seed) * 2.0 - 1.0
    ph = rand01(i, 4, seed) * np.float32(2 * np.pi)
    s = np.sqrt(np.maximum(0.0, 1.0 - z * z))
    d = np.stack([s * np.cos(ph), z, s * np.sin(ph)], axis=1).astype(np.float32)
    sel = rand01(i, 5, seed)
    d[sel < axis_parallel_fraction, 0] = 0.0
    m2 = (sel >= axis_parallel_fraction) & (sel < 1.5 * axis_parallel_fraction)
    d[m2, 1] = 0.0
    d[m2, 2] = -0.0
    m3 = (sel >= 1.5 * axis_parallel_fraction) & (sel < 2.0 * axis_parallel_fraction)
    d[m3, 0] = np.float32(1e-9)  # below FLT_EPSILON -> treated as axis-parallel by vsafe_inverse
    bad = (d * d).sum(axis=1) < 1e-12
    d[bad] = (0, 0, -1)
    rays = np.zeros(n, RAY_DTYPE)
    rays["org"] = o.astype(np.float32)
    rays["dir"] = d
    rays["min_t"] = np.float32(1e-3)
    diag = float(np.linalg.norm(bmax - bmin))
    finite = rand01(i, 6, seed) < 0.5
    mt = np.full(n, 1e30, np.float32)
    mt[finite] = (rand01(i, 7, seed)[finite] * np.float32(diag)).astype(np.float32)
    rays["max_t"] = mt
    return rays
