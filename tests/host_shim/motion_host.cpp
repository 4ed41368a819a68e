// csrc/env_core.cuh's obstacle_run (the moving obstacles' run(), uavrl_env_set_motion) compiled for the host: advances a table
// of n rows (x, y, vx, vy) by `steps` runs.  Built with -ffp-contract=off like the product's host code.
#include "../../dqn-based-uav-3d_path_planer_b200/csrc/env_core.cuh"

extern "C" void shim_obstacle_run(int n, double *rows, double len, double width, int steps)
{
    for (int s = 0; s < steps; ++s)
        for (int i = 0; i < n; ++i) {
            uavrl::MoveObs o{ rows[4 * i], rows[4 * i + 1], rows[4 * i + 2], rows[4 * i + 3] };
            uavrl::obstacle_run(o, len, width);
            rows[4 * i] = o.x; rows[4 * i + 1] = o.y; rows[4 * i + 2] = o.vx; rows[4 * i + 3] = o.vy;
        }
}
