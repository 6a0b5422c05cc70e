"""TEST INFRASTRUCTURE -- generate tests/golden/curved.npz from the LIVE, unmodified reference (imported through
oracle/ref_shim.py, whose strict-interior stub stands in for shapely).

Run in the build container only:   python oracle/gen_curved_golden.py

Curved environments built from many short walls, as the reference's README and its successor-features demo make them:
  circle    the README's arena, a 100-vertex boundary of radius 0.5 (100 walls; linspace(0, 2 pi, 100) repeats its first
            vertex up to rounding, so wall 99 is 1.2e-16 m long, at (0.5, 0))
  annulus   the demo's loop track: that circle with a 100-vertex hole of radius 0.4 (200 walls)
Per environment, in the shape of gen_golden.gen_polygon: a seeded native 1000-step run (Agent, Euclidean PlaceCells,
BVCs) with the default PlaceCells' wall geometry, 384 teacher-forced single steps (half of them started 2-20 mm from
an edge at speed, some at the closing edge), PlaceCells / BVC get_state at those positions, and sample_positions.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from gen_golden import GOLD, mode_a  # noqa: E402


def circle(r, n=100):
    return [[r * np.cos(t), r * np.sin(t)] for t in np.linspace(0, 2 * np.pi, n)]


CASES = (("circle", {"boundary": circle(0.5)}),
         ("annulus", {"boundary": circle(0.5), "holes": [circle(0.4)]}))


def main():
    riab = ref_shim.import_reference()
    assert riab is not None, "reference not present"
    from ratinabox.Environment import Environment
    from ratinabox.Agent import Agent
    from ratinabox.Neurons import PlaceCells, BoundaryVectorCells
    out = {}
    for name, params in CASES:
        np.random.seed(29)
        Env = Environment(dict(params))
        Ag = Agent(Env, {"dt": 0.02, "speed_mean": 0.25})
        PCs = PlaceCells(Ag, {"n": 24, "widths": 0.1, "wall_geometry": "euclidean"})
        BVCs = BoundaryVectorCells(Ag, {"n": 6})
        out[f"{name}_walls"] = Env.walls.copy()
        out[f"{name}_extent"] = np.array(Env.extent, dtype=float)
        out[f"{name}_pos0"], out[f"{name}_vel0"] = Ag.pos.copy(), Ag.velocity.copy()
        out[f"{name}_centres"], out[f"{name}_widths"] = PCs.place_cell_centres.copy(), PCs.place_cell_widths.copy()
        out[f"{name}_bvc"] = np.stack((BVCs.tuning_distances, BVCs.tuning_angles, BVCs.sigma_distances, BVCs.sigma_angles))
        st = np.random.get_state()
        out[f"{name}_rng_keys"], out[f"{name}_rng_pos"], out[f"{name}_rng_has_gauss"], out[f"{name}_rng_cached"] = st[1], st[2], st[3], st[4]
        for _ in range(1000):
            Ag.update(); PCs.update(); BVCs.update()
        out[f"{name}_pos"], out[f"{name}_vel"] = np.array(Ag.history["pos"]), np.array(Ag.history["vel"])
        out[f"{name}_pc_fr"], out[f"{name}_bvc_fr"] = np.array(PCs.history["firingrate"]), np.array(BVCs.history["firingrate"])
        inside = all(Env.check_if_position_is_in_environment(p) for p in out[f"{name}_pos"])
        np.random.seed(4)
        out[f"{name}_default_geom"] = np.array(PlaceCells(Ag, {"n": 4}).wall_geometry)
        print(f"curved[{name}]: {len(Env.walls)} walls, default geometry {out[f'{name}_default_geom']}, trajectory inside: {inside}")
        # mode A single steps: random positions, half of them 2-20 mm from an edge moving at speed, and a few at the
        # closing edge of the boundary (wall n_boundary - 1 between the first vertex and its rounded repeat)
        rs = np.random.RandomState(5)
        A = 384
        np.random.seed(77)
        pos0 = Env.sample_positions(n=A, method="random")
        ang = rs.uniform(0, 2 * np.pi, size=A)
        vel0 = rs.rayleigh(0.4, size=A)[:, None] * np.stack((np.cos(ang), np.sin(ang)), axis=1)
        wl = Env.walls
        for a in range(A // 2):                                 # near an edge, heading at it within +-60 degrees
            w = wl[rs.randint(len(wl))]
            q = w[0] + rs.uniform(0.05, 0.95) * (w[1] - w[0])
            nrm = np.array([-(w[1] - w[0])[1], (w[1] - w[0])[0]])
            if np.linalg.norm(nrm) < 1e-9:
                continue
            nrm /= np.linalg.norm(nrm)
            for sgn in (1.0, -1.0):
                cand = q + sgn * rs.uniform(0.002, 0.02) * nrm
                if Env.check_if_position_is_in_environment(cand):
                    pos0[a] = cand
                    phi = np.arctan2(-sgn * nrm[1], -sgn * nrm[0]) + rs.uniform(-np.pi / 3, np.pi / 3)
                    vel0[a] = rs.uniform(0.5, 1.5) * np.array([np.cos(phi), np.sin(phi)])
                    break
        for k, a in enumerate(range(A // 2, A // 2 + 16)):       # towards the closing edge at (0.5, 0), from both sides
            pos0[a] = [0.5 - rs.uniform(0.002, 0.02), (k - 7.5) * 1e-3]
            vel0[a] = [rs.uniform(0.3, 0.8), rs.uniform(-0.1, 0.1)]
        xi = rs.normal(size=(A, 2))
        outp, outv, outmv = [], [], []
        for a in range(A):
            Ag.pos, Ag.velocity = pos0[a].copy(), vel0[a].copy()
            Ag.rotational_velocity, Ag.measured_velocity = 0.0, vel0[a].copy()
            Ag.head_direction, Ag.distance_travelled = vel0[a] / np.linalg.norm(vel0[a]), 0.0
            with mode_a(list(xi[a])):
                Ag.update()
            outp.append(Ag.pos.copy()); outv.append(Ag.velocity.copy()); outmv.append(Ag.measured_velocity.copy())
        out[f"{name}_A_pos0"], out[f"{name}_A_vel0"], out[f"{name}_A_xi"] = pos0, vel0, xi
        out[f"{name}_A_pos"], out[f"{name}_A_vel"], out[f"{name}_A_mv"] = np.array(outp), np.array(outv), np.array(outmv)
        bounced = int((np.abs(np.linalg.norm(np.array(outv), axis=1) - 0.5 * 0.25) < 1e-12).sum())
        print(f"curved[{name}] mode A: {bounced} / {A} steps bounced")
        with mode_a([]):
            out[f"{name}_A_pc"] = PCs.get_state(evaluate_at=None, pos=pos0)
            out[f"{name}_A_bvc"] = BVCs.get_state(evaluate_at=None, pos=pos0)
        np.random.seed(3)
        out[f"{name}_samples_uj"] = Env.sample_positions(n=50, method="uniform_jitter")
        np.random.seed(8)
        out[f"{name}_samples_random"] = Env.sample_positions(n=500, method="random")
    np.savez_compressed(os.path.join(GOLD, "curved.npz"), **out)
    print("curved.npz", os.path.getsize(os.path.join(GOLD, "curved.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
