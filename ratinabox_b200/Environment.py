"""Host mirror of ``ratinabox.Environment`` for the CUDA step engine.

Only what the hot path needs lives here (SURVEY.md section 8): a 2D environment -- the rectangular
box (solid or periodic) or a polygon ``boundary`` with optional ``holes`` (solid) -- with internal walls.
Construction semantics follow the reference: boundary walls first, in the reference's corner order
(ratinabox/Environment.py:118-144), then the ``walls`` param, the walls of the holes (:147-160), and
later ``add_wall`` calls in insertion order (:330-342).  Anything outside that (1D, objects) raises
``NotImplementedError`` instead of silently taking a different path.
"""
import copy
import warnings

import numpy as np


class Environment:
    default_params = {            # ratinabox/Environment.py:65-75
        "dimensionality": "2D",
        "boundary_conditions": "solid",
        "scale": 1,
        "aspect": 1,
        "dx": 0.01,
        "boundary": None,
        "walls": [],
        "holes": [],
        "objects": [],
    }

    def __init__(self, params={}):
        self.params = copy.deepcopy(__class__.default_params)
        self.params.update(params)
        unexpected = [k for k in params if k not in __class__.default_params]
        if unexpected:                                              # utils.check_params, utils.py:877-916
            warnings.warn(f"Found {len(unexpected)} unexpected params key(s) while initializing Environment: {unexpected}")
        for k, v in self.params.items():
            setattr(self, k, v)
        if self.dimensionality != "2D":
            raise NotImplementedError("ratinabox_b200 accelerates 2D environments only (SURVEY.md section 2 row 9)")
        if self.boundary_conditions not in ("solid", "periodic"):
            raise ValueError(f"unknown boundary_conditions {self.boundary_conditions!r}")
        self.D = 2
        self.Agents = []
        self.agents_dict = {}
        if self.boundary is None:                                   # Environment.py:112-125
            self.is_rectangular = True
            self.boundary = [[0, 0], [self.aspect * self.scale, 0], [self.aspect * self.scale, self.scale], [0, self.scale]]
        else:
            self.is_rectangular = False
        b = self.boundary
        user_walls = np.array(self.walls, dtype=float).reshape(-1, 2, 2)
        if self.boundary_conditions == "periodic" and not self.is_rectangular:      # Environment.py:129-135
            # the reference warns and only rewrites params["boundary_conditions"]: the attribute stays "periodic" and
            # no boundary walls are built -- that combination is outside the hot path
            raise NotImplementedError("periodic boundary conditions need the rectangular box (Environment.py:129-135)")
        if self.boundary_conditions == "solid":                     # Environment.py:137-144
            boundary_walls = np.array([[b[(i + 1) if (i + 1) < len(b) else 0], b[i]] for i in range(len(b))], dtype=float)
            self.walls = np.vstack((boundary_walls, user_walls))
            self.n_boundary_walls = len(b)
        else:                                                       # periodic: no boundary walls are built
            self.walls = user_walls
            self.n_boundary_walls = 0
        self.has_holes = len(self.holes) > 0                        # Environment.py:146-160
        self.hole_wall0, self.n_hole_walls = len(self.walls), 0     # the hole walls are walls[hole_wall0 : +n_hole_walls]
        if self.has_holes:
            assert np.array(self.holes).ndim == 3, ("Incorrect dimensionality for holes list. It must be a list of "
                                                    "lists of coordinates")
            if self.boundary_conditions != "solid":
                raise NotImplementedError("holes need solid boundary conditions")
            for h in self.holes:
                hole_walls = np.array([[h[(i + 1) if (i + 1) < len(h) else 0], h[i]] for i in range(len(h))], dtype=float)
                self.walls = np.vstack((self.walls, hole_walls))
                self.n_hole_walls += len(h)
        self.is_polygonal = (not self.is_rectangular) or self.has_holes
        self.passed_in_objects = copy.deepcopy(self.objects)         # Environment.py:175-187
        self.objects = {"objects": np.empty((0, self.D)), "object_types": np.empty(0, int)}
        self.n_object_types = 0
        self.object_colormap = "rainbow_r"
        for o in self.passed_in_objects:
            self.add_object(o, type=0)
        left, right = min(c[0] for c in b), max(c[0] for c in b)
        bottom, top = min(c[1] for c in b), max(c[1] for c in b)
        self.centre = np.array([(left + right) / 2, (top + bottom) / 2])
        self.extent = np.array([left, right, bottom, top], dtype=float)
        self.discrete_coords = self.discretise_environment(dx=self.dx)
        self.flattened_discrete_coords = self.discrete_coords.reshape(-1, self.discrete_coords.shape[-1])
        self._walls_version = 0
        self._dev = {}          # device -> (version, tensor)

    @property
    def los_skip(self):
        """How many leading walls the line_of_sight / geodesic distances ignore: the reference hard-codes
        ``walls[4:]`` (Environment.py:715-717) whatever the boundary polygon's vertex count."""
        return 0 if self.boundary_conditions == "periodic" else min(4, len(self.walls))

    # ------------------------------------------------------------------ registry
    def add_agent(self, agent=None):                                # Environment.py:220-250
        if agent.name in self.agents_dict:
            raise ValueError(f"An agent with the name {agent.name} already exists in the environment.")
        self.Agents.append(agent)
        self.agents_dict[agent.name] = agent

    # --------------------------------------------------------------------- walls
    def add_wall(self, wall):                                       # Environment.py:330-342
        wall = np.asarray(wall, dtype=float).reshape(1, 2, 2)
        self.walls = np.concatenate((self.walls, wall), axis=0)
        self._walls_version += 1

    def add_object(self, object, type="new"):                        # Environment.py:366-395
        object = np.array(object, dtype=float).reshape(1, -1)
        assert object.shape[1] == self.D
        if type == "new":
            type = self.n_object_types
        elif type == "same":
            type = 0 if len(self.objects["object_types"]) == 0 else self.objects["object_types"][-1]
        else:
            assert type <= self.n_object_types, (
                f"Newly added object must be one of the existing types (currently {np.unique(self.objects['object_types'])}) "
                f"or the next one along ({self.n_object_types}), not {type}")
        type = np.array([type], int)
        self.objects["objects"] = np.append(self.objects["objects"], object, axis=0)
        self.objects["object_types"] = np.append(self.objects["object_types"], type, axis=0)
        self.n_object_types = len(np.unique(self.objects["object_types"]))

    def _walls_signature(self):
        return (self._walls_version, self.walls.shape[0], hash(self.walls.tobytes()))

    def walls_device(self, device):
        """(W,2,2) float64 walls on ``device`` (re-uploaded when they changed)."""
        import torch
        sig = self._walls_signature()
        hit = self._dev.get(device)
        if hit is None or hit[0] != sig:
            t = torch.as_tensor(np.ascontiguousarray(self.walls, dtype=np.float64), device=device)
            self._dev[device] = (sig, t)
            return t
        return hit[1]

    # ------------------------------------------------------------------ sampling
    def sample_positions(self, n=10, method="uniform_jitter"):      # Environment.py:560-633 (2D)
        ex = self.extent
        if method == "random":
            positions = np.zeros((n, 2))
            positions[:, 0] = np.random.uniform(ex[0], ex[1], size=n)
            positions[:, 1] = np.random.uniform(ex[2], ex[3], size=n)
            if self.is_polygonal:                                   # :592-600 brute-force resampling
                # one vectorised test of the n draws, then the reference's draw order: each outside point, in index
                # order, re-drawn by its own sample_positions(n=1) call
                for i in np.flatnonzero(~self._in_environment(positions)):
                    positions[i] = self.sample_positions(n=1, method="random").reshape(-1)
            return positions
        if method[:7] == "uniform":
            area = (ex[1] - ex[0]) * (ex[3] - ex[2])
            if self.has_holes:
                area -= sum(_polygon_area(h) for h in self.holes)
            delta = np.sqrt(area / n)
            x = np.linspace(ex[0] + delta / 2, ex[1] - delta / 2, int((ex[1] - ex[0]) / delta))
            y = np.linspace(ex[2] + delta / 2, ex[3] - delta / 2, int((ex[3] - ex[2]) / delta))
            positions = np.array(np.meshgrid(x, y)).reshape(2, -1).T
            if self.is_polygonal:                                   # :612-615 drop the illegal grid points
                positions = positions[self._in_environment(positions)]
            n_uniform = positions.shape[0]
            if method[7:] == "_jitter":
                positions = positions + np.random.uniform(-0.45 * delta, 0.45 * delta, positions.shape)
            n_remaining = n - n_uniform
            if n_remaining > 0:
                extra = np.array([positions[i] for i in np.random.choice(range(len(positions)), n_remaining, replace=True)])
                delta /= 2
                extra = extra + np.random.uniform(-0.45 * delta, 0.45 * delta, extra.shape)
                positions = np.vstack((positions, extra))
            return positions
        raise ValueError(f"unknown sampling method {method!r}")

    def discretise_environment(self, dx=None):                      # Environment.py:635-655
        dx = self.dx if dx is None else dx
        minx, maxx, miny, maxy = self.extent
        self.x_array = np.arange(minx + dx / 2, maxx, dx)
        self.y_array = np.arange(miny + dx / 2, maxy, dx)[::-1]
        xm, ym = np.meshgrid(self.x_array, self.y_array)
        return np.stack((xm, ym), axis=-1)

    def check_if_position_is_in_environment(self, pos):             # Environment.py:781-818
        pos = np.asarray(pos, dtype=float).reshape(-1)
        if not self.is_polygonal:
            e = self.extent
            return bool((pos[0] > e[0]) and (pos[0] < e[1]) and (pos[1] > e[2]) and (pos[1] < e[3]))
        is_in = _polygon_contains_strict(self.boundary, pos)        # shapely `contains`: strict interior
        for h in self.holes:
            is_in = is_in and not _polygon_contains_strict(h, pos)
        return bool(is_in)

    def _in_environment(self, positions):
        """check_if_position_is_in_environment of every row of an (m, 2) array of a polygonal environment, as a bool
        array: the same float64 decisions as the scalar test (which a few points take: it is faster there, and
        sample_positions re-draws outside points one at a time)."""
        if len(positions) <= 4:
            return np.array([self.check_if_position_is_in_environment(p) for p in positions], dtype=bool)
        is_in = _polygon_contains_strict_many(self.boundary, positions)
        for h in self.holes:
            is_in &= ~_polygon_contains_strict_many(h, positions)
        return is_in


def _polygon_contains_strict(verts, p):
    """Even-odd ray cast; points on an edge or a vertex are NOT inside (shapely ``contains``,
    Environment.py:810-817).  Same arithmetic as ``edges_contain`` in csrc/riab_motion.cuh."""
    x, y = float(p[0]), float(p[1])
    n = len(verts)
    inside = False
    for i in range(n):
        x0, y0 = float(verts[i][0]), float(verts[i][1])
        x1, y1 = float(verts[(i + 1) % n][0]), float(verts[(i + 1) % n][1])
        cross = (x1 - x0) * (y - y0) - (y1 - y0) * (x - x0)
        if cross == 0.0 and min(x0, x1) <= x <= max(x0, x1) and min(y0, y1) <= y <= max(y0, y1):
            return False
        if (y0 > y) != (y1 > y):
            xi = x0 + (y - y0) * (x1 - x0) / (y1 - y0)
            if x < xi:
                inside = not inside
    return inside


def _polygon_contains_strict_many(verts, points):
    """_polygon_contains_strict of every row of an (m, 2) array: the same float64 operations in the same order, one
    edge at a time over all points, so every decision equals the scalar one."""
    pts = np.asarray(points, dtype=float).reshape(-1, 2)
    x, y = pts[:, 0], pts[:, 1]
    n = len(verts)
    inside = np.zeros(len(pts), dtype=bool)
    on_edge = np.zeros(len(pts), dtype=bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(n):
            x0, y0 = float(verts[i][0]), float(verts[i][1])
            x1, y1 = float(verts[(i + 1) % n][0]), float(verts[(i + 1) % n][1])
            cross = (x1 - x0) * (y - y0) - (y1 - y0) * (x - x0)
            on_edge |= (cross == 0.0) & (min(x0, x1) <= x) & (x <= max(x0, x1)) & (min(y0, y1) <= y) & (y <= max(y0, y1))
            straddles = (y0 > y) != (y1 > y)                 # implies y1 != y0: the division below is only used there
            xi = x0 + (y - y0) * (x1 - x0) / (y1 - y0)
            inside ^= straddles & (x < xi)
    return inside & ~on_edge


def _polygon_area(verts):
    v = np.asarray(verts, dtype=float)
    return 0.5 * abs(np.dot(v[:, 0], np.roll(v[:, 1], -1)) - np.dot(v[:, 1], np.roll(v[:, 0], -1)))
