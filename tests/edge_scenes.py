"""Seeded inputs built directly in numpy (not through the synthetic lidar) that sit on the edges where the kernels'
exactness arguments are decided: rank-deficient map neighbourhoods, exact float distance boundaries, duplicated and
dense map points, kilometre offsets, and residual-block sets that end the trust-region solve in each of its ways."""
import numpy as np

F32 = np.float32
ONE_BELOW = np.nextafter(F32(1.0), F32(0.0))          # 1 - 2^-24, the largest float32 below 1


def _pts(xyz, intensity=0.0):
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    out = np.zeros((len(xyz), 4), F32)
    out[:, :3] = xyz
    out[:, 3] = intensity
    return out


def sqdist_f32(p, q):
    """((dx*dx)+(dy*dy))+(dz*dz) in float32, the order every k-NN of the project (and FLANN's L2_Simple) uses"""
    d = (np.asarray(p, F32)[..., :3] - np.asarray(q, F32)[..., :3]).astype(F32)
    return ((d[..., 0] * d[..., 0]) + (d[..., 1] * d[..., 1])) + (d[..., 2] * d[..., 2])


def map_sites():
    """Named five-point (or larger) neighbourhoods, each at least 3 m from every other, with one query per site placed
    so that its five nearest map points are the site's own.  Returns [(name, points (n, 4) f32, queries (m, 4) f32)]."""
    xs = np.linspace(0.1, 0.5, 5)
    sites = []

    def add(name, pts, queries=None):
        pts = _pts(pts)
        if queries is None:
            queries = pts[:, :3].astype(np.float64).mean(0)
        sites.append((name, pts, _pts(queries)))

    # collinear along x (rank 2): Eigen pivots z then x and drops y -> plane z = 2; unpivoted QR fits a different plane
    add("line_x_y1_z2", np.stack([xs, np.ones(5), np.full(5, 2.0)], 1))
    # collinear at negative x (rank 2): unpivoted QR hits R_33 == 0 exactly -> a NaN normal that passes the 0.2 m test
    add("line_x_y12", np.stack([np.linspace(-7.3, -6.6, 5), np.full(5, 12.0), np.full(5, 1.5)], 1))
    # collinear, 1 m long (rank 2): without the rank cut-off both the pivoted and the unpivoted QR divide by ~0
    add("line_x_3to4", np.stack([np.linspace(3.0, 4.0, 5), np.full(5, 0.5), np.full(5, -2.0)], 1))
    # nearly collinear: one point 1e-3 m and ~1e-6 m (float32-rounded) off the line -> full rank, ill-conditioned
    p = np.stack([np.linspace(20.0, 20.4, 5), np.full(5, 5.0), np.full(5, 3.0)], 1); p[2, 1] += 1e-3
    add("near_line_1e-3", p)
    p = np.stack([np.linspace(30.0, 30.4, 5), np.full(5, 5.0), np.full(5, 3.0)], 1); p[2, 1] += 1e-6
    add("near_line_1e-6", p)
    # coplanar through the origin (rank 2: the z column is 0, or the x and y columns are equal)
    add("plane_z0", [[-3.2, -3.1, 0], [-2.8, -3.3, 0], [-3.0, -2.7, 0], [-3.3, -2.9, 0], [-2.9, -2.9, 0]])
    add("plane_x_eq_y", [[-10.0, -10.0, 0.1], [-10.2, -10.2, -0.1], [-9.8, -9.8, 0.2], [-10.1, -10.1, 0.3], [-9.9, -9.9, -0.2]])
    # one point five times (rank 1) and eight times (ties on (distance, index) beyond the fifth neighbour)
    add("dup5", np.tile([15.0, -6.0, 1.0], (5, 1)))
    add("dup8", np.tile([15.0, -12.0, 1.0], (8, 1)), [[15.0, -12.0, 1.0], [15.125, -12.0, 1.0]])
    # isotropic in a plane (corner fit: ev[2] == ev[1] -> no line) and a clean line along (1,1,0) for contrast
    add("cross", [[5.0, 25.0, 5.0], [5.3, 25.0, 5.0], [4.7, 25.0, 5.0], [5.0, 25.3, 5.0], [5.0, 24.7, 5.0]])
    t = np.linspace(-0.3, 0.3, 5)
    add("diag_line", np.stack([5.0 + t, 35.0 + t, np.full(5, 5.0)], 1), [[5.0, 35.0, 5.0]])
    # fifth neighbour at float d^2 == 1.0 exactly (rejected: sqd[4] < 1.0 is false) ...
    q = np.array([40.0, 0.0, 0.0])
    add("d2_one", [q + [0.0625, 0, 0], q + [0, 0.0625, 0], q + [0, 0, 0.0625], q + [0, 0, -0.0625], q + [1.0, 0, 0]], [q])
    # ... and at 1 - 2^-24, the largest float below 1 (accepted): dx = 1 - 2^-24, dy = 2^-12 around x = 0 (both sides of cell 0)
    q = np.array([-0.5, 30.0, 0.0])
    far = [float(F32(0.5) - F32(2.0 ** -24)), 30.0 + 2.0 ** -12, 0.0]
    add("d2_below_one", [q + [0.0625, 0, 0], q + [0, 0.0625, 0], q + [0, 0, 0.0625], q + [0, 0, -0.0625], far], [q])
    return sites


def dense_block(rng, centre, n=2000, half=0.75):
    """n uniform points in a cube of edge 2*half: more than 27 x 32 points in one 27-cell block (several warp rounds)"""
    return _pts(np.asarray(centre) + rng.uniform(-half, half, (n, 3)))


def around_cell_zero(rng, n=400):
    """points on both sides of 0 in every axis, and queries at -0.0, +-1 ulp and exact cell edges"""
    pts = _pts(rng.uniform(-1.6, 1.6, (n, 3)) + [0, 0, 60.0])
    tiny = float(np.nextafter(F32(0), F32(1)))
    qs = _pts([[-0.0, -0.0, 60.0], [tiny, -tiny, 60.0], [-tiny, tiny, 60.0], [1.0, -1.0, 61.0], [-1.0, 1.0, 59.0],
               [0.5, -0.5, 60.5], [-1e-7, 1e-7, 60.0]])
    return pts, qs


def map_scene(seed=0):
    """(map (n, 4) f32, queries (m, 4) f32, site of each map point, site name of each query): every site, a dense block
    and a cloud around cell 0; 'dense' / 'cell0' queries have no fixed neighbour set"""
    rng = np.random.default_rng(seed)
    pts, qs, pid, qname = [], [], [], []
    for name, p, q in map_sites():
        pts.append(p); qs.append(q); pid += [name] * len(p); qname += [name] * len(q)
    d = dense_block(rng, [60.0, 60.0, 10.0])
    pts.append(d); pid += ["dense"] * len(d)
    qs.append(_pts(rng.uniform(-0.7, 0.7, (40, 3)) + [60.0, 60.0, 10.0])); qname += ["dense"] * 40
    c, cq = around_cell_zero(rng)
    pts.append(c); pid += ["cell0"] * len(c)
    qs.append(cq); qname += ["cell0"] * len(cq)
    return np.concatenate(pts), np.concatenate(qs), np.array(pid), np.array(qname)


# ------------------------------------------------------------------------------------------------ residual blocks


def quat(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([np.sin(angle / 2) * axis, [np.cos(angle / 2)]])


def rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def blocks(orc, rng, x_true, n, noise=0.0, kinds=(0, 1, 2), s_values=(1.0,), extent=20.0):
    """n residual blocks cycling through `kinds` (0 edge, 1 plane, 2 plane-norm) whose minimum is x_true up to `noise`
    (metres, on the target geometry).  Edge and plane blocks take their interpolation ratio from `s_values` in turn;
    the target is placed with the pose applied at that ratio, so s != 1 blocks are consistent only for s = 1."""
    R = rot(x_true[:4])
    out = []
    for i in range(n):
        kind = kinds[i % len(kinds)]
        s = s_values[i % len(s_values)]
        cp = rng.uniform(-extent, extent, 3)
        w = R @ cp + x_true[4:] + rng.normal(0, noise, 3) if noise else R @ cp + x_true[4:]
        if kind == 0:
            d = rng.normal(0, 1, 3); d /= np.linalg.norm(d)
            out.append(orc.make_edge(cp, w + 0.5 * d, w - 0.7 * d, s))
        elif kind == 1:
            u = rng.normal(0, 1, 3); v = rng.normal(0, 1, 3)
            out.append(orc.make_plane(cp, w, w + u, w + v, s))
        else:
            nv = rng.normal(0, 1, 3); nv /= np.linalg.norm(nv)
            out.append(orc.make_plane_norm(cp, nv, -float(nv @ w)))
    return np.array(out).reshape(-1, orc.BLOCK_DOUBLES)


def near_parallel_planes(orc, seed, n=30):
    """plane-norm blocks whose normals lie within ~3 degrees of z, for a pose rotated 0.5-2.5 rad about a near-x axis:
    translation in x / y and yaw are barely constrained, so the Gauss-Newton step of the 1e4 initial radius overshoots
    and the solve rejects steps (radius shrinks, decrease factor doubles) from the identity start"""
    rng = np.random.default_rng(seed)
    xt = np.concatenate([quat([1, 0.2, 0], rng.uniform(0.5, 2.5)), [rng.uniform(-5, 5), 0, 0]])
    R = rot(xt[:4])
    out = []
    for _ in range(n):
        cp = rng.uniform(-30, 30, 3)
        w = R @ cp + xt[4:] + rng.normal(0, 0.3, 3)
        nv = np.array([0, 0, 1.0]) + rng.normal(0, 0.05, 3); nv /= np.linalg.norm(nv)
        out.append(orc.make_plane_norm(cp, nv, -float(nv @ w)))
    return np.array(out)


# ------------------------------------------------------------------------------------------------ scan-to-scan search


def ring_major(xyz, rings, frac=0.05):
    """(n, 4) float32 cloud sorted by ring (stable), intensity = ring + frac, the layout of a "last" cloud"""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    rings = np.asarray(rings)
    order = np.argsort(rings, kind="stable")
    out = _pts(xyz[order])
    out[:, 3] = (rings[order] + frac).astype(F32)
    return out


def bucket_of(x, y, nb=128):
    """azimuth bucket of the odometry index (float32 atan2 -- can differ from the device's atan2f by one ulp, so
    callers keep their points away from bucket edges)"""
    a = np.arctan2(np.asarray(y, F32), np.asarray(x, F32)).astype(F32)
    return np.clip(((a + F32(np.pi)) * F32(nb / (2 * np.pi))).astype(np.int32), 0, nb - 1)


def search_clouds(rng, width=64):
    """non-lidar clouds for k-NN: {name: (cloud, queries)}, rings drawn from 0 .. width - 1 (the dense cells on rings 5 and
    width - 24)"""
    out = {}
    n = 3000
    xyz = rng.uniform(-20, 20, (n, 3))
    q = np.concatenate([rng.uniform(-20, 20, (400, 3)), [[0, 0, 0], [0, 0, 7.5], [0, 0, -3], [-5, 0.0, 1], [-5, -0.0, 1],
                                                         [-12, -0.0, -2], [1e-30, 0, 0]]])
    out["uniform"] = (ring_major(xyz, rng.integers(0, width, n)), _pts(q))
    out["one_point"] = (ring_major([[3.0, -4.0, 0.5]], [17]), _pts(rng.uniform(-30, 30, (50, 3))))
    # everything at one azimuth, queries on the opposite side: the sweep must go round the whole circle
    phi = rng.uniform(0.30, 0.31, 400); rho = rng.uniform(3, 4, 400)
    c = np.stack([rho * np.cos(phi), rho * np.sin(phi), rng.uniform(-1, 1, 400)], 1)
    phq = rng.uniform(0.3, 0.31, 40) + np.pi; rq = rng.uniform(2, 8, 40)
    out["one_azimuth"] = (ring_major(c, rng.integers(0, width, 400)),
                          _pts(np.stack([rq * np.cos(phq), rq * np.sin(phq), rng.uniform(-1, 1, 40)], 1)))
    # dense cells: 40 and 1000 points in one (bucket, ring) cell, plus copies of points on other rings
    d1 = np.stack([10 + rng.uniform(0, 0.05, 40), rng.uniform(0, 0.05, 40), rng.uniform(0, 0.05, 40)], 1)
    d2 = np.stack([-10 + rng.uniform(0, 0.05, 1000), 3 + rng.uniform(0, 0.05, 1000), rng.uniform(0, 0.05, 1000)], 1)
    dup = np.repeat(d1[:5], 3, axis=0)
    xyz = np.concatenate([d1, d2, dup]); rings = np.concatenate([np.full(40, 5), np.full(1000, width - 24), np.repeat([6, 7, 8], 5)])
    qd = np.concatenate([d1 + rng.normal(0, 0.01, d1.shape), d2[:200] + rng.normal(0, 0.01, (200, 3)), d1[:5]])
    out["dense_cells"] = (ring_major(xyz, rings), _pts(qd))
    return out


def assoc_scene(seed=0, width=64):
    """A "last" corner / surf cloud (ring-major) of isolated sites in the sweep-start frame, and the start-frame positions
    of the queries meant for them.  Sites:
      tie    closest point A on ring rc; exact copies of one point B on rings rc+1 and rc-1 (2nd point: forward against
             backward), and C on ring rc just before and just after A (same-ring forward against backward), copies of A on
             ring rc+1 at every fourth site (1st point: index order; elsewhere the 2nd point ties)
      far    points whose query lies 8.5-10 deg (3-3.5 buckets) away at 9-12 m (bucket-by-bucket growth)
      wrap   points at azimuth pi - 0.05 with their queries at -pi + 0.004 (the interval wraps past +-pi)
      near   sites at 2-5 m (the rho < 6.5 m first interval)
      edge   sites on rings 0 and width - 1 only (clamped ring slices), and at width 128 also on rings 64 and 63 (either side
             of the middle of the ring range)
    Rings are those of a context of `width` rings (64, or 128 above 64 rings).  Returns (corner_last, surf_last, queries_start_frame (m, 3) float64, tags)."""
    rng = np.random.default_rng(seed)
    pts, rings, q, tags = [], [], [], []

    def site(a, rc, tag, with_ties=True, offset=None):
        a = np.asarray(a, np.float64)
        rho = np.hypot(a[0], a[1]); ux, uy = a[0] / rho, a[1] / rho
        tang = np.array([-uy, ux, 0.0])
        # the site's points along the tangent (a line for corner fits, a plane patch with the up direction for surf fits)
        if with_ties:
            b = a + [0, 0, 0.25]
            c = a + 0.2 * tang + [0, 0, 0.0625]
            up, dn = min(rc + 1, width - 1), max(rc - 1, 0)
            P = [a - 0.3 * tang, c, a, c, a + 0.3 * tang, b, b]; R = [rc, rc, rc, rc, rc, up, dn]
            if with_ties == "first":                       # a copy of A on the next ring: the 1st point ties instead
                P.append(a); R.append(up)
        else:                                              # no copies; one point on the next ring makes a correspondence
            P = [a - 0.3 * tang, a, a + 0.3 * tang, a + [0, 0, 0.25]]; R = [rc, rc, rc, min(rc + 1, width - 1)]
        pts.extend(P); rings.extend(R)
        q.append(a + (offset if offset is not None else rng.normal(0, 0.02, 3))); tags.append(tag)

    for k in range(24):                                    # tie sites all round the circle, 12-20 m
        phi = -np.pi + (k + 0.5) * 2 * np.pi / 24
        rho = rng.uniform(12, 20)
        site([rho * np.cos(phi), rho * np.sin(phi), rng.uniform(-2, 2)], int(rng.integers(2, width - 2)), "tie",
             with_ties="first" if k % 4 == 3 else True)
    for k in range(6):                                     # queries 2-3 buckets from their only neighbours
        phi = 0.2 + k * 0.9; rho = rng.uniform(9, 12); dphi = np.deg2rad(rng.uniform(8.5, 10.0))
        a = np.array([rho * np.cos(phi), rho * np.sin(phi), 0.5])
        qpos = np.array([rho * np.cos(phi + dphi), rho * np.sin(phi + dphi), 0.5])
        site(a, 30 + k, "far", with_ties=False, offset=qpos - a)
    for k in range(4):                                     # across +-pi
        rho = 8 + 2 * k
        a = np.array([rho * np.cos(np.pi - 0.05), rho * np.sin(np.pi - 0.05), -1.0 + k])
        qpos = np.array([rho * np.cos(-np.pi + 0.004), rho * np.sin(-np.pi + 0.004), -1.0 + k])
        site(a, 10 + k, "wrap", offset=qpos - a)
    for k in range(6):
        phi = 1.0 + k * 0.7; rho = 2 + 0.5 * k
        site([rho * np.cos(phi), rho * np.sin(phi), -0.5], 20 + k, "near")
    edge = [width - 1, 0, width - 1, 0] + ([64, 63] if width > 64 else [])
    for k, rc in enumerate(edge):
        phi = -2.5 + k * 0.3
        site([15 * np.cos(phi), 15 * np.sin(phi), 3.0], rc, "edge")
    cloud = ring_major(pts, rings)
    return cloud, cloud.copy(), np.array(q), np.array(tags)


def to_current_frame(p_start, q, t, rings, frac=0.05):
    """points of the current sweep whose TransformToStart (q p + t, s = 1) is p_start: p = q^-1 (p_start - t)"""
    R = rot(q)
    cur = (np.asarray(p_start) - t) @ R       # R^T (p - t) for row vectors
    out = _pts(cur)
    out[:, 3] = (np.asarray(rings) + frac).astype(F32)
    return out


# ------------------------------------------------------------------------------------------------ ring features

_ROOM = np.array([[8.0, 1.0], [4.0, 9.0], [-6.0, 7.5], [-9.0, -1.0], [-3.0, -8.0], [7.0, -6.5]])   # convex, around 0


def _room_range(phi, verts):
    """horizontal range from the origin to the polygon along azimuth phi (vectorised)"""
    d = np.stack([np.cos(phi), np.sin(phi)], 1)
    best = np.full(len(phi), np.inf)
    for i in range(len(verts)):
        a, b = verts[i], verts[(i + 1) % len(verts)]
        e = b - a
        den = d[:, 0] * (-e[1]) - d[:, 1] * (-e[0])
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (a[0] * (-e[1]) - a[1] * (-e[0])) / den
            u = (d[:, 0] * a[1] - d[:, 1] * a[0]) / den
        ok = (t > 0) & (u >= -1e-12) & (u <= 1 + 1e-12)
        best = np.where(ok & (t < best), t, best)
    return best


def vlp16_elevation(ring):
    return -15.0 + 2.0 * ring                    # beam centres of scanRegistration.cpp's N_SCANS == 16 formula


def ring_elevation(ring, n_scans=16):
    """degrees at the middle of `ring` of the elevation formula of n_scans (scanRegistration.cpp:166-205); for 64 rings the upper
    block holds rings 0..32 and the lower block rings 33..50 (ring 0 and the block change sit on a decision: keep them empty)"""
    if n_scans == 16:
        return vlp16_elevation(ring)
    if n_scans == 32:
        return -92.0 / 3.0 + (4.0 * ring + 2.0) / 3.0
    return 2.0 - ring / 3.0 if ring <= 32 else -8.83 - (ring - 32) / 2.0


DENSE_STYLES = ("smooth", "zigzag", "dyadic")
DENSE_STEP = 0.1    # metres between consecutive returns of a smooth or zigzag arc (the suppression break is sqrt(0.05) = 0.224 m)


def dense_arc(n, phi, dist, style, z=0.0, el=None):
    """n returns in firing order (clockwise) on a wall `dist` metres away across azimuth phi, consecutive returns less than
    0.22 m apart, so that a pick marks 5 positions on either side -- a pole, a person or a car close to a beam that sees
    nothing else.  style:
      smooth  a concave corner: two walls at +-20 deg meeting at phi, 0.1 m steps (flat points, sharp ones at the corner)
      zigzag  the same with the range alternating by +-6.25 cm (every point a corner candidate)
      dyadic  a straight wall 0.125 m steps, its second half zigzagging by +-6.25 cm, coordinates multiples of 2^-10 m; with
              phi in {0, +-pi/2} and constant z, equal geometry gives bit-equal curvatures (ties at 0 and at 0.5625)
    z: height of every return; el (degrees): z = horizontal range * tan(el) instead (elevation-mode rings)."""
    u = np.array([np.cos(phi), np.sin(phi)])
    t = np.array([np.sin(phi), -np.cos(phi)])                     # clockwise along the wall
    k = np.arange(n)
    if style == "dyadic":
        s = (k - n // 2) * 0.125
        off = np.where(k >= n // 2, np.where(k % 2 == 0, 0.0625, -0.0625), 0.0)
        xy = dist * u + s[:, None] * t + off[:, None] * u
    else:
        s = (k - (n - 1) / 2.0) * DENSE_STEP
        xy = dist * u + s[:, None] * t - (np.abs(s) * np.tan(np.deg2rad(20.0)))[:, None] * u
        if style == "zigzag":
            xy = xy + np.where(k % 2 == 0, 0.0625, -0.0625)[:, None] * u
    zz = np.hypot(xy[:, 0], xy[:, 1]) * np.tan(np.deg2rad(el)) if el is not None else np.full(n, float(z))
    p = np.concatenate([xy, zz[:, None]], 1)
    if style == "dyadic":
        p = np.round(p * 1024.0) / 1024.0
    return p


def _dense_place(r, style):
    """azimuth and wall distance of ring r's dense arc: spread round the sweep, away from its start and end at +-pi"""
    if style == "dyadic":
        return (np.pi / 2, 0.0, -np.pi / 2)[r % 3], 4.0 + r % 4
    return -2.4 + 4.8 * ((0.618034 * r) % 1.0), 3.5 + (r % 5) * 0.75


def _arc_key(p, r):
    """fraction of the clockwise turn from azimuth pi at which a sensor fires the returns p of ring r"""
    return (np.pi - np.arctan2(p[:, 1], p[:, 0])) / (2 * np.pi) + r * 1e-9


def _firing_order(parts):
    """[(xyz (n, 3), firing key (n,), ring value)] -> (n, 4) float32 in firing order, float 3 = the ring value"""
    xyz = np.concatenate([p for p, _, _ in parts])
    key = np.concatenate([k for _, k, _ in parts])
    out = _pts(xyz)
    out[:, 3] = np.concatenate([np.full(len(p), v, np.float64) for p, _, v in parts])
    return out[np.argsort(key, kind="stable")]


def room_scan(counts, dyadic=False, zigzag=(), far=(), shift=(0.0, 0.0), scale=1.0, dense=(), dense_style="smooth", n_scans=16):
    """A VLP-16 scan of a polygon room (walls meeting at corners: sharp features), points in firing order.
    counts[r] = returns of ring r (0 allowed).  zigzag: rings whose range alternates by +-0.0625 m (a two-letter
    curvature alphabet: every point is a corner candidate, picks crowd the segment boundaries).  far: (ring, first,
    count, range_m) blocks of consecutive returns on a wall `range_m` away.  dyadic: coordinates rounded to 2^-10 m, so
    that equal geometry gives bit-equal curvatures.  dense: rings whose returns lie on a dense arc (dense_arc, in
    `dense_style`) instead of the whole turn.  n_scans: 32 / 64 put ring r at the middle of that elevation formula's ring."""
    verts = _ROOM * scale - np.asarray(shift)
    parts = []
    for r, n in enumerate(counts):
        if n == 0:
            continue
        el = ring_elevation(r, n_scans)
        if r in dense:
            phi, dist = _dense_place(r, dense_style)
            p = dense_arc(n, phi, dist * scale, dense_style, el=el)
            key = _arc_key(p, r)
            if dyadic:
                p = np.round(p * 1024.0) / 1024.0
            parts.append((p, key, 0.0))
            continue
        k = np.arange(n)
        phi = np.pi - 2.0 * np.pi * (k + 0.37) / n                   # clockwise: -atan2(y, x) increases
        rho = _room_range(phi, verts)
        if r in zigzag:
            rho = rho + np.where(k % 2 == 0, 0.0625, -0.0625)
        for ring, first, cnt, rng_m in far:
            if ring == r:
                rho[first:first + cnt] = rng_m
        p = np.stack([rho * np.cos(phi), rho * np.sin(phi), rho * np.tan(np.deg2rad(el))], 1)
        if dyadic:
            p = np.round(p * 1024.0) / 1024.0
        parts.append((p, (k + 0.37) / n + r * 1e-9, 0.0))
    return _firing_order(parts)


def short_ring_scan(counts, style, shift=(0.0, 0.0)):
    """A field-mode scan (ring id in float 3, aloam_config.ring_source = ALOAM_RING_FIELD): ring r holds counts[r] returns;
    rings of fewer than 64 returns lie on a dense arc (dense_arc; style = one of DENSE_STYLES, or one per ring), the others
    take the whole turn of the polygon room.  Heights are constant per ring.  shift: the sensor's position in the room
    (rounded to 2^-10 m, so that dyadic arcs stay dyadic)."""
    shift = np.round(np.asarray(shift, np.float64) * 1024.0) / 1024.0
    parts = []
    for r, n in enumerate(counts):
        if n == 0:
            continue
        st = style if isinstance(style, str) else style[r]
        z = np.round((-2.0 + 3.0 * r / len(counts)) * 1024.0) / 1024.0
        if n < 64:
            phi, dist = _dense_place(r, st)
            p = dense_arc(n, phi, dist, st, z=z)
            p[:, :2] -= shift
            parts.append((p, _arc_key(p, r), float(r)))
        else:
            k = np.arange(n)
            phi = np.pi - 2.0 * np.pi * (k + 0.37) / n
            rho = _room_range(phi, _ROOM - shift)
            parts.append((np.stack([rho * np.cos(phi), rho * np.sin(phi), np.full(n, z)], 1), (k + 0.37) / n + r * 1e-9, float(r)))
    return _firing_order(parts)


def suppression_reach(full):
    """per point of a ring-major cloud: how many neighbours forward / backward a pick marks (scanRegistration.cpp's
    squared-distance > 0.05 break), in float32"""
    p = full[:, :3].astype(F32)
    d = p[1:] - p[:-1]
    step = ((d[:, 0] * d[:, 0]) + (d[:, 1] * d[:, 1])) + (d[:, 2] * d[:, 2])      # step[i] = |p[i+1] - p[i]|^2
    n = len(p)
    rf = np.zeros(n, int); rb = np.zeros(n, int)
    for i in range(n):
        for l in range(1, 6):
            if i + l >= n or step[i + l - 1] > 0.05:
                break
            rf[i] = l
        for l in range(1, 6):
            if i - l < 0 or step[i - l] > 0.05:
                break
            rb[i] = l
    return rb, rf
