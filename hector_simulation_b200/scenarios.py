"""Synthetic robot-state batches for the five BASELINE.json configs (SURVEY.md §8d).

Everything here is *harness*: it restates, in numpy, the cheap host-side data preparation that the
reference's caller performs before it reaches the C boundary, so that the records fed to the
solver look like what ``ConvexMPCLocomotion::updateMPCIfNeeded`` would produce:

  * contact table      Gait::mpc_gait            ConvexMPC/GaitGenerator.cpp:85-103
  * foot positions     leg forward kinematics    src/common/LegController.cpp:108-113,190-194
                       hip offsets               include/common/Biped.h:9-24
  * joint-angle chain  (quirk Q7: offsets added in LegController.cpp:111-113 and again in
                        ConvexMPCLocomotion.cpp:298-313 before the boundary)
  * r, weights, traj   ConvexMPCLocomotion.cpp:315-406

Output records use the reference's ``update_data_t`` layout (convexMPC_interface.h:19-37).
"""
from __future__ import annotations

import numpy as np

K_MAX_GAIT_SEGMENTS = 36

UPDATE_DTYPE = np.dtype(
    [
        ("p", "<f4", 3), ("v", "<f4", 3), ("q", "<f4", 4), ("w", "<f4", 3), ("r", "<f4", 6),
        ("joint_angles", "<f4", 10), ("yaw", "<f4"), ("weights", "<f4", 12),
        ("traj", "<f4", 12 * K_MAX_GAIT_SEGMENTS), ("Alpha_K", "<f4", 12),
        ("gait", "u1", K_MAX_GAIT_SEGMENTS), ("hack_pad", "u1", 1000), ("max_iterations", "<i4"),
        ("rho", "<f8"), ("sigma", "<f8"), ("solver_alpha", "<f8"), ("terminate", "<f8"),
    ],
    align=True,
)
assert UPDATE_DTYPE.itemsize == 3016

# ConvexMPCLocomotion.cpp:321-322
MPC_WEIGHTS = np.array([100, 100, 250, 200, 200, 300, 1, 1, 1, 1, 1, 1], dtype=np.float64)
MPC_ALPHA = np.array([1e-4, 1e-4, 5e-4, 1e-4, 1e-4, 5e-4, 1e-2, 1e-2, 1e-2, 1e-2, 1e-2, 1e-2], dtype=np.float64)
DT_MPC = 0.001 * 40  # FSMState_Walking.cpp:5, ConvexMPCLocomotion.cpp:20
F_MAX = 500.0        # ConvexMPCLocomotion.cpp:410
MU_PASSED = 0.25     # ConvexMPCLocomotion.cpp:410 (ignored by the solver, quirk Q3)
BODY_HEIGHT = 0.55   # ConvexMPCLocomotion.cpp:54


def mpc_gait(n_segments: int, offsets, durations, iteration: int) -> np.ndarray:
    """Contact table [n_segments*2] of 0/1, order [step][leg] (GaitGenerator.cpp:85-103)."""
    table = np.zeros(n_segments * 2, dtype=np.int32)
    for i in range(n_segments):
        it = (i + iteration) % n_segments
        for j in range(2):
            progress = it - offsets[j]
            if progress < 0:
                progress += n_segments
            table[i * 2 + j] = 1 if progress < durations[j] else 0
    return table


def walking_table(horizon: int, iteration: int) -> np.ndarray:
    # walking(horizonLength, (0,5), (5,5))  ConvexMPCLocomotion.cpp:16, scaled with the horizon for N != 10
    half = horizon // 2
    return mpc_gait(horizon, (0, half), (half, horizon - half), iteration)


def standing_table(horizon: int) -> np.ndarray:
    # standing(horizonLength, (0,0), (10,10))  ConvexMPCLocomotion.cpp:17
    return mpc_gait(horizon, (0, 0), (horizon, horizon), 0)


def rpy_to_quat(rpy) -> np.ndarray:
    """ZYX Euler -> (w,x,y,z), body-to-world (what Gazebo's model_states carries)."""
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2), np.sin(y / 2)
    return np.array([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy,
                     cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy])


def quat_to_R(q) -> np.ndarray:
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def quat_to_rpy(q) -> np.ndarray:
    # include/common/Math/orientation_tools.h:208-221
    a = min(2.0 * (q[2] * q[0] - q[1] * q[3]), 1.00001)
    a = max(min(a, 1.0), -1.0)
    return np.array([np.arctan2(2 * (q[0] * q[1] + q[2] * q[3]), 1 - 2 * (q[1] ** 2 + q[2] ** 2)),
                     np.arcsin(a),
                     np.arctan2(2 * (q[0] * q[3] + q[1] * q[2]), 1 - 2 * (q[2] ** 2 + q[3] ** 2))])


def hip_yaw_location(leg: int) -> np.ndarray:
    # Biped.h:11-13,19-22
    return np.array([-0.005, -0.057 if leg == 0 else 0.057, -0.126])


def leg_fk(q, leg: int) -> np.ndarray:
    """Foot position in the hip frame, LegController.cpp:190-194; q already carries the first
    0.3/-0.6/0.3 * 3.14159 offset (LegController.cpp:111-113)."""
    q0, q1, q2, q3, q4 = q
    side = 1.0 if leg == 0 else -1.0
    s, c = np.sin, np.cos
    x = (-(3 * c(q0)) / 200
         - (9 * s(q4) * (c(q3) * (c(q0) * c(q2) - s(q0) * s(q1) * s(q2)) - s(q3) * (c(q0) * s(q2) + c(q2) * s(q0) * s(q1)))) / 250
         - (11 * c(q0) * s(q2)) / 50 - (side * s(q0)) / 50
         - (11 * c(q3) * (c(q0) * s(q2) + c(q2) * s(q0) * s(q1))) / 50
         - (11 * s(q3) * (c(q0) * c(q2) - s(q0) * s(q1) * s(q2))) / 50
         - (9 * c(q4) * (c(q3) * (c(q0) * s(q2) + c(q2) * s(q0) * s(q1)) + s(q3) * (c(q0) * c(q2) - s(q0) * s(q1) * s(q2)))) / 250
         - (23 * c(q1) * side * s(q0)) / 1000 - (11 * c(q2) * s(q0) * s(q1)) / 50)
    y = ((c(q0) * side) / 50
         - (9 * s(q4) * (c(q3) * (c(q2) * s(q0) + c(q0) * s(q1) * s(q2)) - s(q3) * (s(q0) * s(q2) - c(q0) * c(q2) * s(q1)))) / 250
         - (3 * s(q0)) / 200 - (11 * s(q0) * s(q2)) / 50
         - (11 * c(q3) * (s(q0) * s(q2) - c(q0) * c(q2) * s(q1))) / 50
         - (11 * s(q3) * (c(q2) * s(q0) + c(q0) * s(q1) * s(q2))) / 50
         - (9 * c(q4) * (c(q3) * (s(q0) * s(q2) - c(q0) * c(q2) * s(q1)) + s(q3) * (c(q2) * s(q0) + c(q0) * s(q1) * s(q2)))) / 250
         + (23 * c(q0) * c(q1) * side) / 1000 + (11 * c(q0) * c(q2) * s(q1)) / 50)
    z = ((23 * side * s(q1)) / 1000 - (11 * c(q1) * c(q2)) / 50
         - (9 * c(q4) * (c(q1) * c(q2) * c(q3) - c(q1) * s(q2) * s(q3))) / 250
         + (9 * s(q4) * (c(q1) * c(q2) * s(q3) + c(q1) * c(q3) * s(q2))) / 250
         - (11 * c(q1) * c(q2) * c(q3)) / 50 + (11 * c(q1) * s(q2) * s(q3)) / 50 - 3.0 / 50.0)
    return np.array([x, y, z])


def boundary_inputs(pos, rpy, vel, omega, raw_joints, gait_table, horizon: int = 10,
                    v_des_body=(0.0, 0.0), yaw_rate: float = 0.0, pos_des_err=(0.0, 0.0),
                    roll_pitch_des=(0.0, 0.0), feet_world=None) -> dict:
    """The eleven double-precision arguments of update_problem_data (convexMPC_interface.h:43) that
    the reference's caller would build for this robot state (ConvexMPCLocomotion.cpp:283-406)."""
    pos, rpy, vel, omega = (np.asarray(a, dtype=np.float64) for a in (pos, rpy, vel, omega))
    quat = rpy_to_quat(rpy)
    R = quat_to_R(quat)  # body -> world = rBody^T
    est_rpy = quat_to_rpy(quat)
    # LegController::updateData: first offset (3.14159), FK on the offset angles
    q_leg = np.asarray(raw_joints, dtype=np.float64).reshape(2, 5).copy()
    q_leg[:, 2] += 0.3 * 3.14159
    q_leg[:, 3] -= 0.6 * 3.14159
    q_leg[:, 4] += 0.3 * 3.14159
    if feet_world is None:
        p_foot = [pos + R @ (hip_yaw_location(i) + leg_fk(q_leg[i], i)) for i in range(2)]
    else:  # closed-loop harness: feet pinned in the world
        p_foot = [np.asarray(feet_world[i], dtype=np.float64) for i in range(2)]
    # updateMPCIfNeeded: second offset (3.14159265359) + fmod
    PI = 3.14159265359
    q = q_leg.reshape(10).copy()
    for base in (0, 5):
        q[base + 2] += 0.3 * PI
        q[base + 3] -= 0.6 * PI
        q[base + 4] += 0.3 * PI
    q = np.fmod(q, 2 * PI)
    r = np.array([p_foot[i % 2][i // 2] - pos[i // 2] for i in range(6)])
    yaw = est_rpy[2]
    v_des_world = R @ np.array([v_des_body[0], v_des_body[1], 0.0])
    max_pos_error = 0.05
    x_start = pos[0] + float(np.clip(pos_des_err[0], -max_pos_error, max_pos_error))
    y_start = pos[1] + float(np.clip(pos_des_err[1], -max_pos_error, max_pos_error))
    traj_initial = np.array([roll_pitch_des[0], roll_pitch_des[1], 0.0, x_start, y_start, BODY_HEIGHT,
                             0.0, 0.0, yaw_rate, v_des_world[0], v_des_world[1], 0.0])
    traj = np.zeros(12 * horizon)
    for i in range(horizon):
        traj[12 * i: 12 * i + 12] = traj_initial
        if i == 0:
            traj[0:3] = est_rpy
            traj[3:6] = pos
        else:
            traj[12 * i + 3] = (traj_initial[3] if v_des_world[0] == 0 else pos[0]) + i * DT_MPC * v_des_world[0]
            traj[12 * i + 4] = (traj_initial[4] if v_des_world[1] == 0 else pos[1]) + i * DT_MPC * v_des_world[1]
            traj[12 * i + 2] = traj_initial[2] if yaw_rate == 0 else yaw + i * DT_MPC * yaw_rate
    leg_p = np.array([R.T @ (p_foot[i] - pos) - hip_yaw_location(i) for i in range(2)]) if feet_world is not None \
        else np.array([leg_fk(q_leg[i], i) for i in range(2)])
    return dict(leg_p=leg_p, rpy_est=est_rpy.copy(), wpd=np.array([pos[0] + pos_des_err[0], pos[1] + pos_des_err[1]]),
                state_des=np.array([roll_pitch_des[0], roll_pitch_des[1], v_des_body[0], v_des_body[1], yaw_rate]),
                p_foot=np.array(p_foot), q_leg=q_leg.reshape(10).copy(), rBody=R.T.copy(),  # LegController's angles / world->body (row f-2 inputs)
                p=pos.copy(), v=vel.copy(), q=quat, w=omega.copy(), r=r, joint_angles=q, yaw=float(yaw),
                weights=MPC_WEIGHTS.copy(), state_trajectory=traj, Alpha_K=MPC_ALPHA.copy(),
                gait=np.asarray(gait_table, dtype=np.int32).copy())


def to_record(b: dict, horizon: int, out: np.ndarray | None = None) -> np.ndarray:
    """double -> float narrowing of update_problem_data (convexMPC_interface.cpp:87-99)."""
    rec = np.zeros((), dtype=UPDATE_DTYPE) if out is None else out
    rec["p"], rec["v"], rec["q"], rec["w"], rec["r"] = b["p"], b["v"], b["q"], b["w"], b["r"]
    rec["joint_angles"], rec["yaw"], rec["weights"] = b["joint_angles"], b["yaw"], b["weights"]
    rec["traj"][: 12 * horizon] = b["state_trajectory"]
    rec["Alpha_K"] = b["Alpha_K"]
    rec["gait"][: 2 * horizon] = b["gait"]
    return rec


# numpy mirror of `hmpc_state_t` (include/hector_mpc_b200.h): what updateMPCIfNeeded reads, before any data preparation
STATE_DTYPE = np.dtype([("position", "<f8", 3), ("vWorld", "<f8", 3), ("orientation", "<f8", 4), ("omegaWorld", "<f8", 3),
                        ("rpy", "<f8", 3), ("leg_q", "<f8", 10), ("leg_p", "<f8", 6), ("state_des", "<f8", 5),
                        ("world_position_desired", "<f8", 2), ("gait", "u1", K_MAX_GAIT_SEGMENTS), ("pad", "u1", 4)])
assert STATE_DTYPE.itemsize == 352


# numpy mirror of `hmpc_command_t` (include/hector_mpc_b200.h): the command part of a state, its bytes [256, 312)
COMMAND_DTYPE = np.dtype([("state_des", "<f8", 5), ("world_position_desired", "<f8", 2)])
assert COMMAND_DTYPE.itemsize == 56


def command_candidates(states: np.ndarray, K: int, seed: int) -> np.ndarray:
    """COMMAND_DTYPE [B, K]: K candidate commands per state for hmpc_solve_states_device_multi.  Candidate 0 is the state's
    own command; the others change the body velocity (±0.3 m/s forward, ±0.15 m/s sideways), the yaw rate (±0.4 rad/s) and
    the roll / pitch set-points (±0.05 rad) by seeded uniform amounts, enough to move the optimum and often its active set."""
    rng = np.random.default_rng(seed)
    B = len(states)
    cmd = np.zeros((B, K), COMMAND_DTYPE)
    cmd["state_des"] = states["state_des"][:, None, :]
    cmd["world_position_desired"] = states["world_position_desired"][:, None, :]
    if K > 1:
        scale = np.array([0.05, 0.05, 0.3, 0.15, 0.4])
        cmd["state_des"][:, 1:] += rng.uniform(-1.0, 1.0, (B, K - 1, 5)) * scale
    return cmd


def to_state(b: dict, horizon: int, out: np.ndarray | None = None) -> np.ndarray:
    """The caller-side state of one robot (row f-1 input) for the same tick as `to_record(b)`."""
    st = np.zeros((), dtype=STATE_DTYPE) if out is None else out
    st["position"], st["vWorld"], st["orientation"], st["omegaWorld"] = b["p"], b["v"], b["q"], b["w"]
    st["rpy"], st["leg_q"], st["leg_p"] = b["rpy_est"], b["q_leg"], b["leg_p"].reshape(6)
    st["state_des"], st["world_position_desired"] = b["state_des"], b["wpd"]
    st["gait"][: 2 * horizon] = b["gait"]
    return st


def make_states(inputs, horizon: int = 10) -> np.ndarray:
    out = np.zeros(len(inputs), dtype=STATE_DTYPE)
    for i, b in enumerate(inputs):
        to_state(b, horizon, out[i])
    return out


# numpy mirror of `hmpc_rollout_t` (include/hector_mpc_b200.h): per-robot state of the device-resident closed loop
ROLLOUT_DTYPE = np.dtype([("feet_world", "<f8", 6), ("gait_offset", "<i4", 2), ("gait_duration", "<i4", 2),
                          ("iteration", "<i4"), ("failures", "<i4"), ("iters_total", "<i4"), ("ticks", "<i4")])
assert ROLLOUT_DTYPE.itemsize == 80


def make_rollout(inputs, horizon: int = 10, standing=None, phases=None):
    """-> (states, loop) for hmpc_rollout_device: robot i walks from gait iteration phases[i] (default i mod horizon)
    unless standing[i]; its feet are pinned where `inputs[i]` has them."""
    n = len(inputs)
    loop = np.zeros(n, dtype=ROLLOUT_DTYPE)
    half = horizon // 2
    for i, b in enumerate(inputs):
        loop["feet_world"][i] = np.asarray(b["p_foot"]).reshape(6)
        if standing is not None and standing[i]:
            loop["gait_offset"][i], loop["gait_duration"][i], loop["iteration"][i] = (0, 0), (horizon, horizon), 0
        else:
            loop["gait_offset"][i], loop["gait_duration"][i] = (0, half), (half, horizon - half)
            loop["iteration"][i] = (i % horizon) if phases is None else phases[i]
    states = make_states(inputs, horizon)
    for i in range(n):  # the table must be the one of the loop's iteration counter; a standing robot has no velocity command
        if standing is not None and standing[i]:
            states["state_des"][i] = 0.0
        states["gait"][i, : 2 * horizon] = mpc_gait(horizon, loop["gait_offset"][i], loop["gait_duration"][i], int(loop["iteration"][i]))
    return states, loop


# numpy mirrors of `hmpc_swing_t` / `hmpc_swing_cmd_t` (include/hector_mpc_b200.h): swing-leg controller memory and output
SWING_DTYPE = np.dtype([("p0", "<f8", 6), ("swing_time", "<f8", 2), ("first_swing", "<i4", 2)])
SWING_CMD_DTYPE = np.dtype([("pf", "<f8", 6), ("p_des", "<f8", 6), ("v_des", "<f8", 6), ("q_des", "<f8", 10), ("swing", "<i4", 2)])
assert SWING_DTYPE.itemsize == 72 and SWING_CMD_DTYPE.itemsize == 232


def make_swing(n: int) -> np.ndarray:
    """Fresh swing-controller memory: firstSwing = {true, true} (SwingLegController.h:65)."""
    sw = np.zeros(n, dtype=SWING_DTYPE)
    sw["first_swing"] = 1
    return sw


def gait_phase(iteration_counter, iterations_per_mpc: int, n_iterations: int):
    """Gait::_phase of Gait::setIterations (GaitGenerator.cpp:109-113)."""
    period = iterations_per_mpc * n_iterations
    return (np.asarray(iteration_counter) % period) / float(period)


I_BODY_DIAG = np.array([0.5413, 0.5200, 0.0691])  # RobotState.cpp:45
BODY_MASS = 9.0                                    # SolverMPC.cpp:423


def advance_numpy(states: np.ndarray, loop: np.ndarray, wrench: np.ndarray, status: np.ndarray, horizon: int,
                  dt: float = DT_MPC) -> None:
    """In-place numpy mirror of hmpc_advance_kernel (csrc/hmpc_device.cuh): one closed-loop tick for every robot."""
    N = horizon
    for i in range(len(states)):
        st, lo = states[i], loop[i]
        u = np.asarray(wrench[i][:12], dtype=np.float64)
        lo["failures"] += int((int(status[i]) & 0xFF) != 0)
        lo["iters_total"] += (int(status[i]) >> 8) & 0xFFF
        lo["ticks"] += 1
        pos, vw, ow, rpy = st["position"].copy(), st["vWorld"].copy(), st["omegaWorld"].copy(), st["rpy"].copy()
        R = quat_to_R(st["orientation"])
        feet = lo["feet_world"].reshape(2, 3)
        vdw = R[:, 0] * st["state_des"][2] + R[:, 1] * st["state_des"][3]
        for a in range(2):
            w = st["world_position_desired"][a]
            if w - pos[a] > 0.05:
                w = pos[a] + 0.05
            if pos[a] - w > 0.05:
                w = pos[a] - 0.05
            st["world_position_desired"][a] = w + dt * vdw[a]
        tq = u[6:9] + u[9:12]
        for leg in range(2):
            tq = tq + np.cross(feet[leg] - pos, u[3 * leg: 3 * leg + 3])
        dw = R @ ((R.T @ tq) / I_BODY_DIAG)
        sy, cy, sp, cp = np.sin(rpy[2]), np.cos(rpy[2]), np.sin(rpy[1]), np.cos(rpy[1])
        a0 = (cy * ow[0] + sy * ow[1]) / cp
        a1 = -sy * ow[0] + cy * ow[1]
        a2 = ow[2] + sp * a0
        nrpy = rpy + dt * np.array([a0, a1, a2])
        npos = pos + dt * vw
        nw = ow + dt * dw
        nv = vw + dt * ((u[0:3] + u[3:6]) / BODY_MASS + np.array([0.0, 0.0, -9.81]))
        st["rpy"], st["position"], st["omegaWorld"], st["vWorld"] = nrpy, npos, nw, nv
        # (w,x,y,z) of yaw*pitch*roll, written like the kernel
        sr, cr, spp, cpp, syy, cyy = (np.sin(nrpy[0] / 2), np.cos(nrpy[0] / 2), np.sin(nrpy[1] / 2), np.cos(nrpy[1] / 2),
                                      np.sin(nrpy[2] / 2), np.cos(nrpy[2] / 2))
        q = np.array([cyy * cpp * cr + syy * spp * sr, cyy * cpp * sr - syy * spp * cr,
                      cyy * spp * cr + syy * cpp * sr, syy * cpp * cr - cyy * spp * sr])
        st["orientation"] = q
        R = quat_to_R(q)
        it = int(lo["iteration"]) + 1
        lo["iteration"] = it
        new_table = mpc_gait(N, lo["gait_offset"], lo["gait_duration"], it % N)
        for leg in range(2):
            if st["gait"][leg] == 0 and new_table[leg] == 1:
                hip = hip_yaw_location(leg)
                stance_t = 0.5 * float(lo["gait_duration"][leg]) * dt
                for a in range(2):
                    rel = min(max(nv[a] * stance_t + 0.02 * (nv[a] - vdw[a]), -0.4), 0.4)
                    feet[leg, a] = npos[a] + R[a] @ hip + rel
                feet[leg, 2] = 0.0
        st["gait"][: 2 * N] = new_table
        for leg in range(2):
            st["leg_p"][3 * leg: 3 * leg + 3] = R.T @ (feet[leg] - npos) - hip_yaw_location(leg)


def stand_inputs(horizon: int = 10) -> dict:
    """Config 1: spawn pose, double support (SURVEY.md §8d)."""
    return boundary_inputs((0, 0, BODY_HEIGHT), (0, 0, 0), (0, 0, 0), (0, 0, 0), np.zeros(10),
                           standing_table(horizon), horizon)


def _random_state(rng: np.random.Generator, horizon: int, table, moving: bool) -> dict:
    rpy = rng.normal(0.0, 0.05, 3)
    pos = np.array([0.0, 0.0, BODY_HEIGHT]) + rng.normal(0.0, 0.02, 3)
    vx_cmd = rng.uniform(-0.5, 0.5) if moving else 0.0
    vel = rng.normal(0.0, 0.1, 3) + np.array([vx_cmd, 0.0, 0.0])
    omega = rng.normal(0.0, 0.2, 3)
    joints = rng.normal(0.0, 0.05, 10)
    yaw_rate = rng.uniform(-0.3, 0.3) if (moving and rng.random() < 0.25) else 0.0
    err = rng.normal(0.0, 0.03, 2)
    return boundary_inputs(pos, rpy, vel, omega, joints, table, horizon, v_des_body=(vx_cmd, 0.0),
                           yaw_rate=yaw_rate, pos_des_err=err)


def _stress_state(rng: np.random.Generator, horizon: int, scale: float) -> dict:
    """A state far outside the operating envelope (perturbations `scale` times the walking batches': tilts of tenths of
    a radian, metres per second, set-point errors of decimetres) under a walking, standing or RANDOM contact table (flight
    phases, single steps of support — update_problem_data accepts any table): many friction / moment / force bounds are
    active at the optimum (60-110 rows against ~12 for a walking robot)."""
    rpy = rng.normal(0.0, 0.06 * scale, 3)
    pos = np.array([0.0, 0.0, BODY_HEIGHT]) + rng.normal(0.0, 0.03 * scale, 3)
    vx = rng.uniform(-0.5, 0.5) * scale
    vel = rng.normal(0.0, 0.2 * scale, 3) + np.array([vx, 0.0, 0.0])
    omega = rng.normal(0.0, 0.3 * scale, 3)
    joints = rng.normal(0.0, 0.08 * scale, 10)
    yaw_rate = rng.uniform(-0.5, 0.5) * scale
    err = rng.normal(0.0, 0.05 * scale, 2)
    mode = int(rng.integers(0, 3))
    if mode == 0:
        table = walking_table(horizon, int(rng.integers(0, horizon)))
    elif mode == 1:
        table = standing_table(horizon)
    else:
        table = (rng.random((horizon, 2)) < 0.6).astype(np.int32).reshape(walking_table(horizon, 0).shape)
        if table.sum() == 0:
            table.flat[0] = 1
    vy = 0.1 * scale * rng.normal()
    return boundary_inputs(pos, rpy, vel, omega, joints, table, horizon, v_des_body=(vx, vy), yaw_rate=yaw_rate, pos_des_err=err)


def make_stress_batch(batch: int, horizon: int, scale: float, seed: int) -> np.ndarray:
    """records[batch] of _stress_state: the robustness workload of tests/golden/stress_referee.npz."""
    rng = np.random.default_rng(seed)
    recs = np.zeros(batch, dtype=UPDATE_DTYPE)
    for i in range(batch):
        to_record(_stress_state(rng, horizon, scale), horizon, recs[i])
    return recs


def config_seed(cfg: int) -> int:
    return 20260923 + cfg


def make_batch(cfg: int, batch: int, horizon: int = 10, seed: int | None = None):
    """-> (records[batch] UPDATE_DTYPE, list of boundary-input dicts).

    cfg 1: stand (every record identical)          cfg 2: walking gait, phase = i mod N
    cfg 3: 25 % stand / 75 % walk, random phase    cfg 4: like 3 at the given horizon
    cfg 5: like 2 (initial states of the closed loop)
    """
    rng = np.random.default_rng(config_seed(cfg) if seed is None else seed)
    recs = np.zeros(batch, dtype=UPDATE_DTYPE)
    inputs = []
    for i in range(batch):
        if cfg == 1:
            b = stand_inputs(horizon)
        elif cfg in (2, 5):
            b = _random_state(rng, horizon, walking_table(horizon, i % horizon), moving=True)
        else:
            if rng.random() < 0.25:
                b = _random_state(rng, horizon, standing_table(horizon), moving=False)
            else:
                b = _random_state(rng, horizon, walking_table(horizon, int(rng.integers(0, horizon))), moving=True)
        to_record(b, horizon, recs[i])
        inputs.append(b)
    return recs, inputs
