"""The launch plan of the level kernel (csrc/launch_plan.h: make_launch_plan), restated in plain Python.

The plan is chosen on the host from the batch size, the grid (SMs x resident CTAs per SM) and the level geometry: one
launch per level with squads of up to 69 CTAs for small batches; for batches of at least grid/4 pairs a coarse segment
with one CTA per pair, fused with up to three slices of the fine levels with squads of g, 2g and 4g CTAs; and the developer
overrides DVO_B200_* on top.  test_launch_plan_host.py checks the C++ against this restatement segment for segment;
test_gpu_launch_plans.py uses it to pick batch sizes and to count the persistent launches of a call on the device.  The
tile geometry is the kernel's (tests/tile_geometry.py).
"""
from tile_geometry import TILE_H, TILE_W
OVERHEAD_TILES = 45.0      # level_squad_size's per-stage overhead, in tile-times
COARSE_TILES = 110         # levels of at most this many tiles take one CTA per pair in a walking plan
KNOBS = ("DVO_B200_NO_WALK", "DVO_B200_NO_FUSE", "DVO_B200_CONTIGUOUS", "DVO_B200_COARSE_TILES", "DVO_B200_TAIL",
         "DVO_B200_STRIPS_PER_CTA", "DVO_B200_FINE_G")
OVERRIDES = [("NO_WALK", "1"), ("NO_FUSE", "1"), ("CONTIGUOUS", "1"),
             ("COARSE_TILES", "0"), ("COARSE_TILES", "40"), ("COARSE_TILES", "400"),
             ("TAIL", "0,0"), ("TAIL", "60,30"), ("TAIL", "180,90"),
             ("STRIPS_PER_CTA", "1"), ("STRIPS_PER_CTA", "3"), ("STRIPS_PER_CTA", "69"),
             ("FINE_G", "1"), ("FINE_G", "4"), ("FINE_G", "8")]


def level_geometry(w, h, levels):
    """(nstrips, nbands, rows) of every pyramid level, level 0 first"""
    out = []
    for _ in range(levels):
        out.append(((h + TILE_H - 1) // TILE_H, (w + TILE_W - 1) // TILE_W, h))
        w, h = w // 2, h // 2
    return out


def level_squad_size(nstrips, nbands, grid, npairs, forced_spc=0):
    best_g, best_cost = 1, -1.0
    for spc in range(1, nstrips + 1):
        g = (nstrips + spc - 1) // spc
        if g > grid:
            continue
        if spc > 1 and (nstrips + spc - 2) // (spc - 1) == g:
            continue
        nsquads = min(grid // g, max(npairs, 1))
        per_squad = npairs / nsquads
        cost = (max(per_squad, 1.0) + (1.2 if npairs > nsquads else 0.0)) * (spc * nbands + OVERHEAD_TILES)
        if forced_spc > 0:
            cost = abs(spc - forced_spc)
        if best_cost < 0 or cost < best_cost - 1e-9:
            best_cost, best_g = cost, g
    return best_g


def segment(geom, first, grid, first_li, nlev, g, pair_begin, npairs, env):
    """one segment of a launch: levels [first_li, first_li + nlev) of the match with squads of g CTAs, the pairs
    [pair_begin, pair_begin + npairs)"""
    levels = [geom[first - first_li - k] for k in range(nlev)]
    return {"first_li": first_li, "nlev": nlev, "g": g, "nsquads": min(grid // g, max(npairs, 1)),
            "strips_per_cta": [-(-s // min(g, s)) for s, _, _ in levels], "pair_begin": pair_begin, "npairs": npairs,
            "hmax": max(h for _, _, h in levels), "cyclic": 0 if "DVO_B200_CONTIGUOUS" in env else 1}


def plan(geom, first, last, grid, n, env=None):
    """groups of levels (coarse to fine), whether the two groups run fused in one launch, the fine slices of a fused launch
    (squad size, first pair, pairs), the number of persistent launches per call and the segments of every launch;
    env: the DVO_B200_* overrides"""
    env = env or {}
    tiles = [s * b for s, b, _ in geom]
    nlev = first - last + 1
    forced = int(env.get("DVO_B200_STRIPS_PER_CTA", 0))
    g_level = [level_squad_size(geom[first - li][0], geom[first - li][1], grid, n, forced) for li in range(nlev)]
    walk = n >= grid // 4 and "DVO_B200_NO_WALK" not in env
    ct = int(env.get("DVO_B200_COARSE_TILES", COARSE_TILES))
    groups, li = [], 0
    while li < nlev:
        G = {"first_li": li, "nlev": 1, "g": g_level[li]}
        if walk:
            coarse = tiles[first - li] <= ct
            if coarse:
                G["g"] = 1
            while li + G["nlev"] < nlev and (tiles[first - li - G["nlev"]] <= ct) == coarse:
                if not coarse:
                    G["g"] = g_level[li + G["nlev"]]       # the finest level of the group decides
                G["nlev"] += 1
        fg = int(env.get("DVO_B200_FINE_G", 0))
        if tiles[first - li] > ct and fg > 0:
            G["g"] = min(fg, grid)
        groups.append(G)
        li += G["nlev"]
    fused = len(groups) == 2 and groups[0]["g"] == 1 and "DVO_B200_NO_FUSE" not in env
    slices = []
    if fused:
        F = groups[1]
        min_strips = min(geom[first - F["first_li"] - k][0] for k in range(F["nlev"]))
        g2, g3 = 2 * F["g"], 4 * F["g"]
        fit2, fit3 = g2 <= min_strips and g2 <= grid, g3 <= min_strips and g3 <= grid
        c2 = int(1.8 * (grid // g2) + 0.5) if fit2 else 0
        c3 = int(1.8 * (grid // g3) + 0.5) if c2 and fit3 else 0
        if "DVO_B200_TAIL" in env:
            a2, a3 = (int(v) for v in env["DVO_B200_TAIL"].split(","))
            c2 = a2 if fit2 else 0
            c3 = a3 if c2 and fit3 else 0
        keep = 2 * (grid // F["g"])                       # the first slice keeps at least two pairs per squad
        if n - c2 - c3 < keep:
            c3 = 0
        if n - c2 < keep:
            c2 = 0
        begin = 0
        for k, c in enumerate((n - c2 - c3, c2, c3)):
            if c > 0:
                slices.append((F["g"] << k, begin, c))
                begin += c
    seg = lambda G, g, b, c: segment(geom, first, grid, G["first_li"], G["nlev"], g, b, c, env)
    if fused:
        segments = [[seg(groups[0], groups[0]["g"], 0, n)] + [seg(groups[1], g, b, c) for g, b, c in slices]]
    else:
        segments = [[seg(G, G["g"], 0, n)] for G in groups]
    return {"groups": groups, "walk": walk, "fused": fused, "slices": slices,
            "launches": 1 if fused else len(groups), "g_level": g_level, "segments": segments}


def shape(p):
    """what distinguishes one plan from another for test_gpu_launch_plans.py: per-level launches, or the squad sizes of the
    fused slices"""
    return ("fused",) + tuple(s[0] for s in p["slices"]) if p["fused"] else ("per-level",)


def boundary_sizes(geom, first, last, grid, nmax=512):
    """the first and the last batch size of every plan shape up to nmax, and 2"""
    out, prev = {2}, None
    for n in range(1, nmax + 1):
        s = shape(plan(geom, first, last, grid, n))
        if s != prev:
            out.add(n)
            if n > 1:
                out.add(n - 1)
        prev = s
    out.add(nmax)
    return sorted(out)


def size_of_shape(geom, first, last, grid, want, nmax=512, pick="middle"):
    """a batch size in the first run of sizes that give plan shape `want`"""
    run = []
    for n in range(1, nmax + 1):
        if shape(plan(geom, first, last, grid, n)) == want:
            run.append(n)
        elif run:
            break
    assert run, f"no batch size up to {nmax} reaches plan {want} at grid {grid}"
    return {"first": run[0], "last": run[-1], "middle": run[len(run) // 2]}[pick]
