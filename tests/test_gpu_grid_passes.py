"""GPU: the stage-0 hash-grid passes row by row against the float64 grid oracle (oracle/grid_oracle.py).

The scatter (n2m_s0_encode_bwd), the TV pass (n2m_s0_tv) and the gather (n2m_s0_encode_fwd) are called through their C entry points
on buffers built here, never through a trainer step.  Every sample is a record (t = 0, 0, 0, int_as_float(k)) whose position is
rays_o[k], the way stage 1 feeds the scatter (stage1.cu), so the test places every sample exactly and fixes the order of the samples
in each warp; it writes M (counters[1]) and the ray-range part boundaries (counters[4..12]) itself.  Tile-image columns 0-2 and 51-63
and every row (and record) in [M, Mcap) hold NaN / inf: the passes must not read them.  The oracle runs with the level scales the
kernels compute (exp2f is ex2.approx under -use_fast_math), read off the device by a calibration scatter (Grid._device_geom).

* Exact probes: cotangents whose (row, column) targets have one nonzero contributor each, so that every gradient-table entry must be
  fp32(w_k * g) bit for bit, placed in same-cell runs of zero-cotangent lanes (run lengths 1-32, runs across warps and tiles, A-B-A
  cells, warps of exactly 20 / 21 runs around the merge threshold) at all 16 levels, at lattice points and at u = 0 / u = 1.
* Dense random cotangents on crafted and marched batches, 1 / 2 / 4 / 8 ray-range parts on forked streams: per row
  |gpu - ref| <= c * n_row * 2^-24 * sum|contrib|, and the same set of nonzero rows.  Passing for every part count means the
  parts change nothing but the order of the fp32 additions.
* found_inf, the TV pass (weights, sample counts, concurrent with the scatter into one table) and the gather (one fp16 ulp, rows it
  must leave alone).
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

import cases
from nerf2mesh_b200 import synthetic as S
from nerf2mesh_b200._lib import call, ptr, stream
from nerf2mesh_b200.stage0 import S0Params, Stage0Config, Stage0Trainer
import oracle.grid_oracle as GO
from oracle.grid_oracle import _level_geom, _row_index, level_offsets

pytestmark = pytest.mark.gpu

L = 16
F32 = np.float32
COL_D, COL_C = 3, 19                      # first density / colour gradient column of a tile-image row
C_SCATTER = 2                             # one rounding per product, one per addition
C_TV = 16                                 # -use_fast_math: approximate lambda / 6 and rsqrtf, a few ulps per contribution
_streams = []


def _forked(n):
    while len(_streams) < n:
        _streams.append(torch.cuda.Stream())
    return _streams[:n]


# ------------------------------------------------------------------------------------------------------------------------------
# geometry: the oracle's expressions
# ------------------------------------------------------------------------------------------------------------------------------
class Grid:
    """Level layout of one hash grid: log2(per-level scale) S, base resolution H, normalising bound, row offsets."""

    def __init__(self, S, H, bound=1.0, offs=None, per_level_scale=None):
        self.S, self.H, self.bound = float(F32(S)), int(H), float(bound)
        if offs is None:
            offs = level_offsets(3, L, per_level_scale or float(np.exp2(self.S)), self.H, 19, False)
        self.offs = np.asarray(offs, dtype=np.int32)
        self.rows = int(self.offs[-1])
        self.offsets = torch.from_numpy(self.offs).cuda()
        self.geom = [_level_geom(l, self.S, self.H, self.offs) for l in range(L)]        # (scale, res, rows)
        self.geom = self._device_geom()

    def _device_geom(self):
        """(scale, res, rows) per level with the scale the kernels use.  Under -use_fast_math exp2f is ex2.approx, which numpy does not
        reproduce bit for bit (test_oracle_golden.py), and a one-ulp scale moves every weight.  A sample at u = (u_x, 0, 0) with
        cotangent 1 at level l has corner weights (1 - fx) / 4 and fx / 4 exactly, fx = frac(fma(u_x, scale, 0.5)): a few scatter
        launches give that FMA at several u_x for every level, and the fp32 scale near numpy's that reproduces all of them is the
        device's."""
        b_ = self.bound
        fmas = [[] for _ in range(L)]                                            # (u_x, fp32 FMA result) per level
        for xv in (b_, 0.5 * b_, 0.25 * b_, 0.0, -0.3 * b_, 0.7 * b_, 0.9 * b_, -0.85 * b_):
            x = np.tile(np.array([xv, -b_, -b_], F32), (L, 1))
            u = self.u_of(x)
            cot = np.zeros((L, 48), F32)
            cot[np.arange(L), np.arange(L)] = 1
            b = Bufs(self, x, cot, table=(torch.zeros(self.rows), torch.zeros(self.rows, 2)))
            b.scatter()
            gt = b.gt[:, 0].cpu().numpy()
            for l in range(L):
                base, crn = self.lattice(u[l:l + 1], l)
                fx = F32(4) * gt[int(crn[0, 1])]
                assert F32(4) * gt[int(crn[0, 0])] == F32(1) - fx, ("calibration", l, xv)
                fmas[l].append((float(u[l, 0]), F32(base[0, 0].item()) + fx))
        geom = []
        for l in range(L):
            scale0, _, rows = self.geom[l]
            cands = [F32(scale0)]
            for _ in range(8):
                cands = [np.nextafter(cands[0], F32(0))] + cands + [np.nextafter(cands[-1], F32(np.inf))]
            fits = [s for s in cands if all(F32(ux * float(s) + 0.5) == pos for ux, pos in fmas[l])]
            assert fits, ("no fp32 scale reproduces the device's lattice positions", l)
            scale = fits[len(fits) // 2]
            geom.append((scale, int(np.ceil(scale)) + 1, rows))
        return geom

    @contextlib.contextmanager
    def oracle(self):
        """the grid oracle with this grid's device level scales"""
        orig = GO._level_geom
        GO._level_geom = lambda level, S, H, offsets: self.geom[level]
        try:
            yield
        finally:
            GO._level_geom = orig

    @classmethod
    def of(cls, cfg, offs=None):
        return cls(np.log2(cfg.per_level_scale), cfg.base_resolution, cfg.bound, offs, cfg.per_level_scale)

    def params(self, lambda_tv=0.0):
        p = S0Params()
        p.bound = p.grid_bound = self.bound
        p.inv_2gb = float(F32(1) / F32(2 * self.bound))
        p.S, p.base_res, p.num_levels, p.lambda_tv = self.S, self.H, L, lambda_tv
        p.max_steps, p.cascades, p.grid_size, p.T_thresh = 1024, 1, 128, 1e-4
        return p

    def u_of(self, x):
        """grid coordinates sample_of gives position x: (x + bound) * fp32(1 / (2 bound)), fp32"""
        x = np.asarray(x, dtype=F32)
        return ((x + F32(self.bound)).astype(F32) * (F32(1) / F32(2 * self.bound))).astype(F32)

    def lattice(self, u, l):
        """base cell [B,3] and global corner rows [B,8] of grid coordinates u [B,3] at level l"""
        scale, res, rows = self.geom[l]
        pos = (torch.as_tensor(np.asarray(u)).double() * float(scale) + 0.5).float()     # FMA u * scale + 0.5
        base = torch.floor(pos).clamp(min=0).to(torch.int64)
        crn = [_row_index(base + torch.tensor([c & 1, (c >> 1) & 1, (c >> 2) & 1]), res, rows, 0, False) for c in range(8)]
        return base, torch.stack(crn, 1) + int(self.offs[l])

    def row_counts(self, u):
        """corner contributions per gradient row, all levels"""
        return sum(torch.bincount(self.lattice(u, l)[1].flatten(), minlength=self.rows) for l in range(L)).double()


# ------------------------------------------------------------------------------------------------------------------------------
# crafted batches
# ------------------------------------------------------------------------------------------------------------------------------
class Layout:
    """A sample stream built run by run.  A run is `n` consecutive samples in one lattice cell of level `l`; a run may carry one
    nonzero-cotangent lane (the probe), whose (row, column) targets at level l are kept disjoint from every other probe's."""
    COLSETS = [(0, 1, 2), (0,), (1,), (2,)]

    def __init__(self, g, seed=0):
        self.g, self.rng = g, np.random.default_rng(seed)
        self.x, self.cot, self.run = [], [], []           # per sample: position, 48 gradient columns, (level, run id)
        self.used = {}                                    # (level, column) -> rows already hit by a probe
        self.nprobe = 0
        self._prev = None                                 # (level, cell) of the last run

    def __len__(self):
        return len(self.x)

    def _span(self, l):
        return int(np.floor(float(self.g.geom[l][0]) + 0.5))    # largest base coordinate of level l

    def _point(self, l, cell, frac):
        scale, b = float(self.g.geom[l][0]), self.g.bound
        u = np.clip((np.asarray(cell, float) + frac - 0.5) / scale, 0.0, 1.0)
        return (u * 2 * b - b).astype(F32)

    def _cell_of(self, x, l):
        return tuple(self.g.lattice(self.g.u_of(x)[None], l)[0][0].tolist())

    def _inside(self, l, cell, n=None):
        """a position (n positions) inside `cell` of level l"""
        out = np.empty((n or 1, 3), F32)
        todo = np.arange(len(out))
        for _ in range(100):
            out[todo] = self._point(l, cell, self.rng.uniform(0.1, 0.9, (len(todo), 3)))
            base = self.g.lattice(self.g.u_of(out[todo]), l)[0].numpy()
            todo = todo[(base != np.asarray(cell)).any(1)]
            if not len(todo):
                return out if n else out[0]
        raise AssertionError(("no interior point", l, cell))

    def _lattice_x(self, l, k):
        """an fp32 position whose FMA k - 0.5 + 0.5 lands exactly on lattice coordinate k of level l, or None"""
        scale, b = float(self.g.geom[l][0]), self.g.bound
        x0 = F32(((k - 0.5) / scale) * 2 * b - b)
        for direction in (np.inf, -np.inf):
            x = x0
            for _ in range(64):
                u = self.g.u_of(x)
                if F32(float(u) * float(scale) + 0.5) == k:
                    return x
                x = np.nextafter(x, F32(direction))
        return None

    def _probe_x(self, l, mode):
        span = self._span(l)
        if mode == "corner0":
            return np.full(3, -self.g.bound, F32)
        if mode == "corner1":
            return np.full(3, self.g.bound, F32)
        cell = self.rng.integers(1, span, 3)
        if mode == "lattice":
            xs = []
            for d in range(3):
                for _ in range(50):
                    v = self._lattice_x(l, int(cell[d]))
                    if v is not None:
                        break
                    cell[d] = self.rng.integers(1, span)
                assert v is not None, ("no lattice point", l)
                xs.append(v)
            return np.array(xs, F32)
        x = self._inside(l, cell)
        if mode in ("u0", "u1"):
            x[0] = F32(-self.g.bound if mode == "u0" else self.g.bound)
        return x

    def free(self, x, l, cols):
        """x's 8 corner rows at level l are distinct and not hit by a probe in any column of `cols`"""
        rows = self.g.lattice(self.g.u_of(x)[None], l)[1][0].tolist()
        return len(set(rows)) == 8 and not any(r in self.used.get((l, c), ()) for c in cols for r in rows)

    def _claim(self, x, l, cols):
        """True (and the rows recorded) when x's 8 corner rows at level l are distinct and free in every column of `cols`"""
        if not self.free(x, l, cols):
            return False
        rows = self.g.lattice(self.g.u_of(x)[None], l)[1][0].tolist()
        for c in cols:
            self.used.setdefault((l, c), set()).update(rows)
        return True

    def _filler_cell(self, l, avoid):
        span = self._span(l)
        while True:
            cell = tuple(int(v) for v in self.rng.integers(1, span, 3))
            if cell not in avoid:
                return cell

    def add_run(self, l, n, probe=None, cols=None, mode="interior", cell=None, x=None):
        """`n` samples in one cell of level l (a random one unless `cell` / the probe's position `x` fixes it).  `probe`: the lane
        (offset in the run) that gets nonzero cotangents in `cols` (0 = density, 1, 2 = colour) of level l.  Returns the cell."""
        prev = self._prev[1] if self._prev and self._prev[0] == l else None
        if probe is not None and x is None:
            cols = cols if cols is not None else self.COLSETS[self.nprobe % 4]
            for _ in range(2000):
                x = self._probe_x(l, mode)
                c = self._cell_of(x, l)
                if c != prev and self._claim(x, l, cols):
                    break
            else:
                raise AssertionError(("no free probe cell", l, mode))
        elif probe is not None:
            assert self._claim(x, l, cols), "probe rows taken"
        if x is not None:
            cell = self._cell_of(x, l)
        elif cell is None:
            cell = self._filler_cell(l, {prev})
        assert cell != prev, "consecutive runs must be different cells"
        rid = len(self.run) and self.run[-1][1] + 1
        xs = self._inside(l, cell, n)
        for i in range(n):
            xi = x if (i == probe and x is not None) else xs[i]
            cot = np.zeros(48, F32)
            if i == probe:
                for c in cols:
                    mag = np.exp2(self.rng.uniform(-6, 6)) * (1 + self.rng.random())
                    cot[l if c == 0 else 16 + 2 * l + (c - 1)] = F32(np.float16(mag * self.rng.choice([-1, 1])))
            self.x.append(xi); self.cot.append(cot); self.run.append((l, rid))
        if probe is not None:
            self.nprobe += 1
        self._prev = (l, cell)
        return cell

    def fill(self, l, n, maxlen=2):
        """n lanes of zero-cotangent runs of length <= maxlen"""
        while n > 0:
            k = min(n, int(self.rng.integers(1, maxlen + 1)))
            self.add_run(l, k)
            n -= k

    def pad_to(self, l, m, mod):
        """one zero-cotangent run until len % mod == m (few runs per warp: the scatter's merge stays on)"""
        n = (m - len(self)) % mod
        if n:
            self.add_run(l, n)

    def arrays(self):
        return np.stack(self.x).astype(F32), np.stack(self.cot).astype(F32)


def hash_collision(lay, l):
    """two cells of hashed level l whose corner-row sets intersect"""
    span = lay._span(l)
    seen = {}
    for _ in range(200):
        cells = lay.rng.integers(1, span, (4096, 3))
        x = np.stack([lay._point(l, c, np.full(3, 0.5)) for c in cells])
        _, rows = lay.g.lattice(lay.g.u_of(x), l)
        for i, rs in enumerate(rows.tolist()):
            for r in set(rs):
                j = seen.get(r)
                if (j is not None and tuple(j[1]) != tuple(cells[i]) and lay.free(j[0], l, (0,)) and lay.free(x[i], l, (1, 2))
                        and lay._cell_of(j[0], l) == tuple(j[1]) and lay._cell_of(x[i], l) == tuple(cells[i])):
                    return j[0], x[i]
            for r in rs:
                seen.setdefault(r, (x[i], tuple(cells[i])))
    raise AssertionError("no colliding cells")


def probe_layout(g, seed=0, key_pairs=False):
    """Exact-probe batch: per level, one warp per (run length 1..32, probe at the run's start / middle / end), lattice, u = 0 / 1 and
    grid-corner probes, A-B-A cells, warps of exactly 20 and 21 runs, runs across a warp and across a tile boundary, and on hashed
    levels two adjacent lanes in different cells whose rows collide (density probe beside colour probe).  `key_pairs`: adjacent
    lanes in cells (512, 0, z) / (0, 1, z), whose merge keys collide when a coordinate gets fewer than 10 bits."""
    lay = Layout(g, seed)
    modes = ["interior"] * 5 + ["lattice", "u0", "u1"]
    for l in range(L):
        for n in range(1, 33):
            for off in sorted({0, n - 1} | ({n // 2} if n in (3, 5, 9, 17, 32) else set())):
                pre = int(lay.rng.integers(0, 32 - n + 1))
                lay.fill(l, pre)
                lay.add_run(l, n, probe=off, mode=modes[lay.nprobe % len(modes)])
                lay.fill(l, 32 - n - pre)
        for mode in ("corner0", "corner1"):
            lay.add_run(l, 1, probe=0, mode=mode)
            lay.fill(l, 31)
        # A-B-A
        lay.fill(l, 5)
        a = lay.add_run(l, 3, probe=1)
        lay.add_run(l, 2)
        lay.add_run(l, 4, cell=a)
        lay.fill(l, 18)
        # exactly 20 and 21 runs (the scatter merges at <= 20)
        for ntwo, none in ((12, 8), (11, 10)):
            lens = [2] * ntwo + [1] * none
            lay.rng.shuffle(lens)
            first2 = lens.index(2)
            for i, k in enumerate(lens):
                lay.add_run(l, k, probe=0 if i == first2 else None)
        # runs across a warp boundary (lanes 28-31 | 0-3), probe on either side, and across a tile boundary
        for off, m, mod in ((1, 28, 32), (5, 28, 32), (2, 124, 128)):
            lay.pad_to(l, m, mod)
            lay.add_run(l, 8, probe=off)
            lay.pad_to(l, 0, 32)
        if g.geom[l][2] == 1 << 19 and (g.geom[l][1] + 1) ** 3 > (1 << 19):
            xa, xb = hash_collision(lay, l)
            lay.add_run(l, 1, probe=0, cols=(0,), x=xa)
            lay.add_run(l, 1, probe=0, cols=(1, 2), x=xb)
            lay.pad_to(l, 0, 32)
        if key_pairs and g.geom[l][1] < 1023 and lay._span(l) > 512:
            for cells in (((512, 0, 7), (0, 1, 7)), ((0, 1, 9), (512, 0, 9)), ((0, 512, 11), (0, 0, 12))):
                lay.add_run(l, 3)
                for k, c in enumerate(cells):
                    x = lay._inside(l, c)
                    lay.add_run(l, 1, probe=0 if k == 0 else None, cols=(0, 1, 2), x=x)
            lay.pad_to(l, 0, 32)
    return lay


# ------------------------------------------------------------------------------------------------------------------------------
# device buffers and launches
# ------------------------------------------------------------------------------------------------------------------------------
def tile_image(rows):
    """[Mcap, 64] fp16 rows -> tile images [ntiles][8 chunks][128 rows][8]"""
    return rows.view(-1, 128, 8, 8).permute(0, 2, 1, 3).contiguous().view(-1)


def untile(t, n):
    return t[: n * 64].view(n // 128, 8, 128, 8).permute(0, 2, 1, 3).reshape(n, 64).float()


def pack_table(dens, col):
    """interleaved {f32 density, half2 colour} entries"""
    R = dens.shape[0]
    raw = torch.empty(R, 8, dtype=torch.uint8)
    raw[:, :4] = dens.float().contiguous().view(torch.uint8).view(R, 4)
    raw[:, 4:] = col.half().contiguous().view(torch.uint8).view(R, 4)
    return raw.view(torch.float32).view(R, 2).cuda()


class Bufs:
    """One batch on the device: records, positions, counters (M, part boundaries), tile image of cotangents, tables."""

    def __init__(self, g, x, cot=None, bounds=None, lambda_tv=0.0, loss_scale=1.0, table=None, Mcap=None, seed=1):
        M = x.shape[0]
        self.g, self.M = g, M
        self.Mcap = Mcap or (M // 128 + 2) * 128
        nan = float("nan")
        xyz = torch.full((self.Mcap, 3), nan)
        xyz[:M] = torch.from_numpy(np.asarray(x, F32))
        recs = torch.full((self.Mcap, 4), nan)
        recs[:M, :3] = 0
        recs[:, 3] = torch.arange(self.Mcap, dtype=torch.int32).view(torch.float32)
        dirs = torch.full((self.Mcap, 3), nan)
        dirs[:M] = torch.tensor([0.0, 0.0, 1.0])
        self.xyz, self.recs, self.dirs = xyz.cuda(), recs.cuda(), dirs.cuda()
        rows = torch.empty(self.Mcap, 64, dtype=torch.float16)
        rows[:, 0:3] = torch.tensor([nan, float("inf"), -float("inf")])
        rows[:, 51:64] = torch.tensor([nan, float("inf"), 65504.0, -float("inf")] * 3 + [nan])
        rows[:M, 3:51] = torch.from_numpy(cot).half() if cot is not None else 0
        rows[M:] = torch.tensor([nan, float("inf")] * 32)
        self.rows = rows
        self.denc = tile_image(rows).cuda()
        self.counters = torch.zeros(16, dtype=torch.int32)
        self.counters[0] = self.counters[1] = M
        self.set_bounds(bounds if bounds is not None else [M * e // 8 for e in range(9)])
        gen = torch.Generator().manual_seed(seed)
        if table is None:
            table = (torch.rand(g.rows, generator=gen) * 2 - 1, (torch.rand(g.rows, 2, generator=gen) * 2 - 1).half())
        self.tab_d, self.tab_c = table
        self.table = pack_table(*table)
        self.ls = torch.tensor([loss_scale, 0, 0, 0, 0, 0, 0, 0], dtype=torch.float32).cuda()
        self.p = g.params(lambda_tv)
        self.gt = torch.zeros(g.rows, 4, device="cuda")

    def set_bounds(self, bounds):
        assert len(bounds) == 9 and bounds[0] == 0 and bounds[8] == self.M and list(bounds) == sorted(bounds)
        self.bounds = list(bounds)
        self.counters[4:13] = torch.tensor(self.bounds, dtype=torch.int32)
        self.counters_d = self.counters.cuda()

    def part(self, k, nparts):
        if nparts == 1:
            return 0, self.M
        return self.bounds[k * 8 // nparts], self.bounds[(k + 1) * 8 // nparts]

    def scatter(self, nparts=1, only=None, gt=None):
        """the parts' scatters, part k on forked stream k (part 0 on the current stream), as the trainer runs them"""
        gt = self.gt if gt is None else gt
        main = torch.cuda.current_stream()
        streams = [main] + _forked(nparts - 1)
        for st in streams[1:]:
            st.wait_stream(main)
        for k, st in enumerate(streams):
            if only is not None and k not in only:
                continue
            with torch.cuda.stream(st):
                call("n2m_s0_encode_bwd", ctypes.byref(self.p), ptr(self.recs), ptr(self.counters_d), self.Mcap, ptr(self.xyz),
                     ptr(self.dirs), ptr(self.denc), ptr(self.table), ptr(self.g.offsets), ptr(gt), ptr(self.ls), k, nparts, stream())
        for st in streams[1:]:
            main.wait_stream(st)

    def tv(self, gt=None):
        call("n2m_s0_tv", ctypes.byref(self.p), ptr(self.recs), ptr(self.counters_d), self.Mcap, ptr(self.xyz), ptr(self.dirs),
             ptr(self.table), ptr(self.g.offsets), ptr(self.gt if gt is None else gt), ptr(self.ls), stream())

    def gather(self, enc, part=0, nparts=1):
        call("n2m_s0_encode_fwd", ctypes.byref(self.p), ptr(self.recs), ptr(self.counters_d), self.Mcap, ptr(self.xyz), ptr(self.dirs),
             ptr(self.table), ptr(self.g.offsets), ptr(enc), part, nparts, stream())

    def found_inf(self):
        torch.cuda.synchronize()
        return self.ls[3].item()


# ------------------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------------------
def cot_levels(cot):
    """[M, 48] gradient columns -> the oracle's [L, M, 3] (density, colour 0, colour 1)"""
    c = torch.from_numpy(np.asarray(cot, F32)).double()
    return torch.stack([c[:, :16], c[:, 16::2], c[:, 17::2]], -1).permute(1, 0, 2).contiguous()


class ScatterRef:
    def __init__(self, g, x, cot):
        u = torch.from_numpy(g.u_of(x))
        G = cot_levels(cot)
        with g.oracle():
            self.ref, _ = GO.grid_encode_backward(G, u, g.offs, g.rows, g.S, g.H)
            self.abs, _ = GO.grid_encode_backward(G.abs(), u, g.offs, g.rows, g.S, g.H)
        self.nrow = g.row_counts(u)

    def tol(self, c=C_SCATTER):
        return c * self.nrow[:, None] * 2.0 ** -24 * self.abs


class TVRef:
    """TV gradient in the loss-scaled domain: lambda inside the unit cube, 10 lambda outside when bound > 1"""

    def __init__(self, g, x, dens, lam, loss_scale):
        x = np.asarray(x, F32)
        u = torch.from_numpy(g.u_of(x))
        outer = (np.abs(x).max(-1) > 1) & (g.bound > 1)
        self.n_in, self.n_out = int((~outer).sum()), int(outer.sum())
        emb = dens.float()[:, None]
        self.ref = torch.zeros(g.rows, dtype=torch.float64)
        w = np.zeros(x.shape[0])
        for sel, lam_g in ((~outer, F32(lam)), (outer, F32(lam) * F32(10))):
            if sel.any():
                with g.oracle():
                    self.ref += GO.grad_total_variation(u[torch.from_numpy(sel)], emb, g.offs, float(lam_g) * loss_scale, g.S, g.H)[:, 0]
                w[sel] = float(F32(float(lam_g) * loss_scale) / F32(6))
        # |w * sum * rsqrt(sq)| <= w * sqrt(6) (at most six differences): a bound on each contribution's magnitude
        centre = torch.stack([g.lattice(u, l)[1][:, 0] for l in range(L)], 1)
        ws = torch.from_numpy(w)[:, None].expand(-1, L)
        self.abs = torch.bincount(centre.flatten(), ws.flatten() * 6 ** 0.5, minlength=g.rows)
        self.nrow = torch.bincount(centre.flatten(), minlength=g.rows).double()

    def tol(self, c=C_TV):
        return c * self.nrow * 2.0 ** -24 * self.abs


def check_rows(gpu, ref, tol, what):
    """per-row bound, identical nonzero set"""
    gpu = gpu.double().cpu()
    err = (gpu - ref).abs()
    bad = err > tol
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        pytest.fail(f"{what}: {int(bad.sum())} entries beyond the bound; first at flat index {i}: gpu {gpu.flatten()[i].item()!r} "
                    f"ref {ref.flatten()[i].item()!r} tol {tol.flatten()[i].item()!r}")
    nz_g, nz_r = gpu != 0, ref != 0
    assert torch.equal(nz_g, nz_r), f"{what}: nonzero sets differ in {int((nz_g != nz_r).sum())} entries"


def check_scatter(b, sref, what, extra_x=None, extra_tol=None):
    gt = b.gt.cpu()
    assert torch.equal(gt[:, 3].view(torch.int32), torch.zeros(b.g.rows, dtype=torch.int32)), f"{what}: .w is not +0"
    ref, tol = sref.ref.clone(), sref.tol()
    if extra_x is not None:
        ref[:, 0] += extra_x
        tol[:, 0] += extra_tol
    check_rows(gt[:, :3], ref, tol, what)


def default_grid(bound=1.0):
    return Grid.of(Stage0Config(bound=bound))


_LAYOUTS = {}


def layout(name):
    """the exact-probe batch of the default grid and of a grid whose levels land on resolutions 1021, 1022, 1023, ..."""
    if name not in _LAYOUTS:
        if name == "default":
            g = default_grid()
            lay = probe_layout(g)
        else:
            g = Grid(0.001, 1021)
            res = [gm[1] for gm in g.geom]
            assert res[:3] == [1021, 1022, 1023]
            lay = probe_layout(g, key_pairs=True)
        x, cot = lay.arrays()
        if len(x) % 128 == 0:
            x, cot = x[:-37], cot[:-37]
        _LAYOUTS[name] = (g, lay, x, cot)
    return _LAYOUTS[name]


def check_runs(g, lay, n):
    """the crafted run structure is what the kernel sees: samples of one run share the level-l cell, consecutive runs differ"""
    u = g.u_of(np.stack(lay.x[:n]))
    bases = np.stack([g.lattice(u, l)[0].numpy() for l in range(L)])          # [L, n, 3]
    lv, rid = np.array(lay.run[:n]).T
    i = np.arange(1, n)
    same_level = lv[1:] == lv[:-1]
    same_cell = (bases[lv[1:], i] == bases[lv[1:], i - 1]).all(-1)
    same_run = rid[1:] == rid[:-1]
    bad = same_level & (same_cell != same_run)
    assert not bad.any(), ("run structure", np.nonzero(bad)[0][:5] + 1)


def boundary_sets(M, seed=0):
    """part boundaries inside tiles, on tile edges and with empty parts"""
    rng = np.random.default_rng(seed + M)
    inside = [0] + sorted(rng.integers(0, M + 1, 7).tolist()) + [M]
    edges = [0] + [min(M, 128 * -(-M * e // 1024)) for e in range(1, 8)] + [M]
    empty = [0, 0, M // 3, M // 3, M // 3, M // 2 + 1, M, M, M]
    return [inside, edges, empty]


# ------------------------------------------------------------------------------------------------------------------------------
# 1. exact probes
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nparts", [1, 8])
@pytest.mark.parametrize("grid", ["default", "res1022"])
def test_scatter_exact_probes(grid, nparts):
    g, lay, x, cot = layout(grid)
    M = len(x)
    check_runs(g, lay, M)
    sref = ScatterRef(g, x, cot)
    nz = sref.ref != 0
    assert int(nz.sum()) > 1000
    expect = sref.ref.float()          # one nonzero contributor per entry (Layout._claim): the exact product rounded once, fp32(w_k * g)
    bounds = boundary_sets(M)[0] if nparts > 1 else None
    b = Bufs(g, x, cot, bounds)
    if nparts > 1:                                         # boundaries inside runs and inside tiles
        assert any(v % 128 for v in b.bounds[1:8])
    b.scatter(nparts)
    gt = b.gt.cpu()
    assert b.found_inf() == 0
    assert torch.equal(gt[:, 3].view(torch.int32), torch.zeros(g.rows, dtype=torch.int32))
    diff = (gt[:, :3] != expect).any(1)
    if diff.any():
        r = int(diff.nonzero()[0])
        lvl = int(np.searchsorted(g.offs, r, side="right") - 1)
        pytest.fail(f"{int(diff.sum())} rows differ; first row {r} (level {lvl}): gpu {gt[r, :3].tolist()} expected {expect[r].tolist()}")


# ------------------------------------------------------------------------------------------------------------------------------
# 2. dense random cotangents, ray-range parts
# ------------------------------------------------------------------------------------------------------------------------------
def random_cot(M, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(M, 48, generator=gen) * torch.exp2(torch.randint(-4, 5, (M, 48), generator=gen).float())).half().float().numpy()


@pytest.mark.parametrize("M", [77, 128, 129, None])
def test_scatter_dense_crafted_parts(M):
    g, lay, x, _ = layout("default")
    x = x[:M] if M else x
    M = len(x)
    cot = random_cot(M, 3)
    sref = ScatterRef(g, x, cot)
    b = Bufs(g, x, cot)
    for bounds in boundary_sets(M):
        b.set_bounds(bounds)
        for nparts in (1, 2, 4, 8):
            b.gt.zero_()
            b.scatter(nparts)
            assert b.found_inf() == 0
            check_scatter(b, sref, f"M={M} nparts={nparts} bounds={bounds}")


def marched(name):
    """positions of a marched batch: cases.MARCH_CASES, or 'converged4096' (bench-sized lego batch, 4096 rays)"""
    if name == "converged4096":
        N = 4096
        cfg = Stage0Config(bound=1.0, num_rays=N, max_samples=N * 256)
        _, bits, _ = S.occupancy_regime("converged")
        ro, rd = cases.rays(N, seed=3)
        noises = torch.rand(N, generator=torch.Generator().manual_seed(5))
    else:
        c = cases.march_case(name)
        N = c["rays_o"].shape[0]
        cfg = Stage0Config(bound=c["bound"], contract=c["contract"], dt_gamma=c["dt_gamma"], num_rays=N, max_samples=N * 1024)
        bits, ro, rd, noises = c["bits"], c["rays_o"], c["rays_d"], c["noises"]
    tr = Stage0Trainer(cfg)
    tr.set_occupancy(bits)
    tr.rays_o.copy_(ro); tr.rays_d.copy_(rd); tr.noises.copy_(noises)
    tr.march()
    torch.cuda.synchronize()
    M = int(tr.counters[1].item())
    assert M > 0 and tr.counters[2].item() == 0
    recs = tr.recs[:M].cpu()
    n = recs[:, 3].contiguous().view(torch.int32).long()
    xyz = (ro[n] + recs[:, :1] * rd[n]).clamp(-cfg.real_bound, cfg.real_bound)
    if cfg.contract:
        mag = xyz.abs().amax(-1, keepdim=True)
        xyz = torch.where(mag > 1, xyz * ((2 - 1 / mag) / mag), xyz)
    g = Grid.of(cfg, tr.offsets.cpu().numpy())
    bounds = tr.counters[4:13].cpu().tolist()
    del tr
    return g, xyz.float().numpy(), bounds


@pytest.mark.parametrize("name", cases.MARCH_CASES + ["converged4096"])
def test_scatter_dense_marched_parts(name):
    g, x, bounds = marched(name)
    M = len(x)
    if name == "converged4096":
        # far more (level group, tile) items than the device holds CTAs at once: the grid-stride walk wraps many times
        props = torch.cuda.get_device_properties(0)
        resident = getattr(props, "max_threads_per_multi_processor", 2048) // 128 * props.multi_processor_count
        assert 12 * ((M + 127) // 128) >= 4 * resident, (M, resident)
    cot = random_cot(M, 4)
    sref = ScatterRef(g, x, cot)
    b = Bufs(g, x, cot, bounds)
    for nparts in (1, 2, 4, 8):
        b.gt.zero_()
        b.scatter(nparts)
        assert b.found_inf() == 0
        check_scatter(b, sref, f"{name} nparts={nparts}")


# ------------------------------------------------------------------------------------------------------------------------------
# 3. found_inf
# ------------------------------------------------------------------------------------------------------------------------------
def test_found_inf_exactly_for_owned_gradient_columns():
    g = default_grid()
    _, _, x, _ = layout("default")
    x = x[:300]
    cot = random_cot(300, 5)
    bounds = [0, 60, 60, 130, 200, 200, 250, 290, 300]       # part 0 of 2: [0, 200), part 1: [200, 300); tile 1 is shared
    b = Bufs(g, x, cot, bounds)
    b.scatter(2)
    assert b.found_inf() == 0                              # garbage columns and rows >= M are not read
    base = b.rows.clone()
    for col in range(3, 51):
        rows = base.clone()
        rows[150 + col, col] = float("inf") if col % 2 else float("nan")
        b.denc.copy_(tile_image(rows).cuda())
        b.ls[3] = 0
        b.scatter(2)
        assert b.found_inf() == 1, f"column {col}"
    # a boundary-tile row of part 1: part 0's launch visits the tile but not the row
    rows = base.clone()
    rows[210, 20] = float("inf")
    b.denc.copy_(tile_image(rows).cuda())
    b.ls[3] = 0
    b.scatter(2, only=[0])
    assert b.found_inf() == 0
    b.scatter(2, only=[1])
    assert b.found_inf() == 1


# ------------------------------------------------------------------------------------------------------------------------------
# 4. TV
# ------------------------------------------------------------------------------------------------------------------------------
LAM = 1e-3
LS = 1024.0


def run_tv(g, x, what, bounds=None):
    b = Bufs(g, x, None, bounds, lambda_tv=LAM, loss_scale=LS)
    b.tv()
    torch.cuda.synchronize()
    tref = TVRef(g, x, b.tab_d, LAM, LS)
    c = b.counters_d.cpu()
    assert (int(c[3]), int(c[15])) == (tref.n_in, tref.n_out), what
    gt = b.gt.cpu()
    assert torch.equal(gt[:, 1:].view(torch.int32), torch.zeros(g.rows, 3, dtype=torch.int32)), f"{what}: TV wrote beyond .x"
    check_rows(gt[:, 0], tref.ref, tref.tol(), what)
    return tref


@pytest.mark.parametrize("name", ["crafted", "garden_cascades", "contract", "lego_converged"])
def test_tv_rows(name):
    if name == "crafted":
        g, _, x, _ = layout("default")
        tref = run_tv(g, x, name)
    else:
        g, x, _ = marched(name)
        tref = run_tv(g, x, name)
        assert tref.n_in > 0
        if name == "contract":
            assert tref.n_out > 0                          # 10 lambda outside the unit cube


def test_tv_weight_and_counts_at_the_unit_cube_face():
    """|x| exactly 1.0 is inside the unit cube, the next float above 1.0 is outside (10 lambda), with bound 2"""
    g = Grid.of(Stage0Config(bound=2.0))
    one, above = F32(1.0), np.nextafter(F32(1.0), F32(2))
    rng = np.random.default_rng(3)
    x = rng.uniform(-1.9, 1.9, (700, 3)).astype(F32)
    for i in range(0, 700, 7):
        x[i, i % 3] = one if i % 2 else -one
        x[i + 1, (i + 1) % 3] = above if i % 2 else -above
        x[i + 2] = x[i + 2] * F32(0.5)
    x[600:640] = x[600]                                    # one same-cell run of 40 samples across a warp boundary
    tref = run_tv(g, x, "face")
    assert tref.n_in > 100 and tref.n_out > 100


def test_scatter_and_tv_concurrent_into_one_table():
    g, _, x, _ = layout("default")
    M = len(x)
    cot = random_cot(M, 6)
    b = Bufs(g, x, cot, boundary_sets(M)[0], lambda_tv=LAM, loss_scale=LS)
    sref = ScatterRef(g, x, cot)
    tref = TVRef(g, x, b.tab_d, LAM, LS)
    main = torch.cuda.current_stream()
    side = _forked(8)[7]
    side.wait_stream(main)
    with torch.cuda.stream(side):
        b.tv()
    b.scatter(2)
    main.wait_stream(side)
    assert b.found_inf() == 0
    check_scatter(b, sref, "scatter + TV", tref.ref, tref.tol())


# ------------------------------------------------------------------------------------------------------------------------------
# 5. gather
# ------------------------------------------------------------------------------------------------------------------------------
def f16_ulp(v):
    e = torch.floor(torch.log2(v.abs().clamp(min=2.0 ** -14)))
    return torch.exp2(e - 10)


@pytest.mark.parametrize("grid", ["default", "res1022"])
def test_gather_within_one_fp16_ulp(grid):
    g, _, x, _ = layout(grid)
    M = len(x)
    b = Bufs(g, x, None, boundary_sets(M)[0])
    u = torch.from_numpy(g.u_of(x))
    with g.oracle():
        d_ref, _ = GO.grid_encode_forward(u, b.tab_d.float()[:, None], g.offs, g.S, g.H)
        c_ref, _ = GO.grid_encode_forward(u, b.tab_c.float(), g.offs, g.S, g.H)      # fp16 table values held as float32
    ref = torch.cat([d_ref[:, :, 0].t(), c_ref.permute(1, 0, 2).reshape(M, 32)], 1)
    nt = (M + 127) // 128
    sentinel = -7.0
    enc = torch.full((b.Mcap * 64,), sentinel, dtype=torch.float16, device="cuda")
    b.gather(enc)
    e = untile(enc, b.Mcap).cpu()
    feat = e[:M, 3:51]
    err = (feat.double() - ref.double()).abs()
    ulp = f16_ulp(ref.double())
    assert (err <= ulp).all(), f"max err / ulp {(err / ulp).max().item():.3f}"
    assert torch.equal(e[:M, 0:3], torch.from_numpy(x).half().float())
    assert torch.equal(e[:M, 51:54], torch.tensor([[0.0, 0.0, 1.0]]).expand(M, 3))
    assert torch.equal(e[:M, 54:], torch.zeros(M, 10))
    assert torch.equal(e[M:nt * 128], torch.zeros(nt * 128 - M, 64))                  # whole batch: the last tile's rows past M are 0
    assert (e[nt * 128:] == sentinel).all()
    # parts: a part writes only the rows it owns, and all parts together give the whole batch's rows
    for nparts in (2, 4, 8):
        for k in range(nparts):
            lo, hi = b.part(k, nparts)
            enc.fill_(sentinel)
            b.gather(enc, k, nparts)
            ek = untile(enc, b.Mcap).cpu()
            own = torch.zeros(b.Mcap, dtype=torch.bool)
            own[lo:hi] = True
            assert (ek[~own] == sentinel).all(), (nparts, k)
            assert torch.equal(ek[own], e[own]), (nparts, k)
