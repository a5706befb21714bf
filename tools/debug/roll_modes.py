"""Debug helper: the fast-motion scenario of test_map_grid_roll_and_drop under the three loop modes."""
import os, sys, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if len(sys.argv) > 1:
    import numpy as np
    from loam_velodyne_b200 import api, synth
    from oracle import pydriver
    np.set_printoptions(precision=5, suppress=True, linewidth=200)
    sc = synth.make_scene(seed=3, extent=160.0)
    lidar = synth.Lidar(16, 600, -15.0, 15.0)
    corner, surf = synth.make_map(sc, 150_000, window=150.0)
    pg, pc = api.Pipeline(), pydriver.best().pipeline()
    pg.seed_map(corner, surf); pc.seed_map(corner, surf)
    for i in range(3):
        pts, rs = synth.make_sweep(sc, lidar, i, v=(30.0, 0.0, 0.0), yaw_rate=0.0)
        _, od_g, aft_g, _ = pg.sweep(pts, rs)
        _, od_c, aft_c, _ = pc.sweep(pts, rs)
        print(sys.argv[1], i, "it", pg.odom.last_iterations(), pg.mapping.last_iterations(), "od", np.abs(od_g - od_c).max(), "aft", np.abs(aft_g - aft_c).max())
        print("   od_g", od_g, "\n   od_c", od_c, "\n   aft_g", aft_g, "\n   aft_c", aft_c)
else:
    for name, env in (("hostloop", {"LOAM_B200_DEVICE_LOOP": "0"}), ("graph", {"LOAM_B200_DEVICE_LOOP": "1"})):
        e = dict(os.environ); e.update(env)
        subprocess.run([sys.executable, __file__, name], env=e)
