// SPDX-License-Identifier: Apache-2.0
//
// hostsim.cpp -- TEST INFRASTRUCTURE. Compiles the kernels' per-robot arithmetic
// (upkie_b200/csrc/sim_core.cuh, __host__ __device__) with g++ so that the fp32
// formulation can be checked against the oracle on machines without a GPU
// (`pytest -m "not gpu"`). Never loaded by the product: upkie_b200/_lib.py
// only opens libupkie_b200.so, which has no CPU path.
#include <cmath>
#include <cstring>
#include <string>

#include "../../upkie_b200/csrc/controllers_core.cuh"
#include "../../upkie_b200/csrc/params.h"

using namespace upkie_b200;

struct HostSim {
  SimParams P;
  int scalar_legs = 0;  // 1: step with the scalar-leg substep instead of the paired one the kernels run
};

// The warp vote of the kernels. g_vote_always: every vote says "some other lane still needs this" - the robot stays
// in the PGS loops for all pgs_iterations trips, as a lane does whose warp-mates converge late; its result must not
// change (per-lane freeze of Bullet's residual rule, sim_pair.cuh).
static int g_vote_always = 0;
static bool any_fn(bool p) { return g_vote_always ? true : p; }

extern "C" {

void* hostsim_create(const UpkieModel* m, const UpkieSimConfig* c) {
  HostSim* h = new HostSim();
  std::string err;
  std::memset(&h->P, 0, sizeof(h->P));
  if (make_sim_params(*m, *c, h->P, err) != 0) { delete h; return nullptr; }
  return h;
}
void hostsim_destroy(void* h) { delete static_cast<HostSim*>(h); }

void hostsim_reset(void* hv, int n, float* state, const float* init, const float* eps, const float* mu) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    reset_robot(h->P, S, init + size_t(i) * UPKIE_INIT_DIM, eps ? eps + size_t(i) * 6 : nullptr,
                mu ? mu[i] : h->P.friction, any_fn, h->P.joint_limits);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

void hostsim_set_vote_always(int on) { g_vote_always = on ? 1 : 0; }

void hostsim_set_scalar_legs(void* hv, int on) { static_cast<HostSim*>(hv)->scalar_legs = on ? 1 : 0; }

void hostsim_step_servos(void* hv, int n, float* state, const float* action, float* obs, const float* eps,
                         const float* mu, uint32_t* err) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    const float* e6 = eps ? eps + size_t(i) * 6 : nullptr;
    const float mui = mu ? mu[i] : h->P.friction;
    const uint32_t e = h->scalar_legs ? step_servo_action<true>(h->P, S, a, e6, mui, any_fn)
                                      : step_servo_action<false>(h->P, S, a, e6, mui, any_fn);
    if (err) err[i] = e;
    for (int j = 0; j < 6; ++j) {
      float* o = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = S.torque[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// the same tick, also returning the body-ground contact record of the last substep ([n][UPKIE_BODY_REC_DIM])
void hostsim_step_servos_rec(void* hv, int n, float* state, const float* action, float* obs, const float* eps,
                             const float* mu, float* rec) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    float* r = rec + size_t(i) * UPKIE_BODY_REC_DIM;
    for (int k = 0; k < UPKIE_BODY_REC_DIM; ++k) r[k] = 0.f;
    step_servo_action<false>(h->P, S, a, eps ? eps + size_t(i) * 6 : nullptr, mu ? mu[i] : h->P.friction, any_fn, r);
    for (int j = 0; j < 6; ++j) {
      float* o = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = S.torque[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

void hostsim_step_gyropod(void* hv, int n, float* state, const float* action, int act_dim, float* obs6,
                          uint8_t* terminated) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    const float a0 = action[size_t(i) * act_dim];
    const float a1 = act_dim > 1 ? action[size_t(i) * act_dim + 1] : 0.f;
    gyropod_action(h->P, S, a0, a1, a);
    if (h->scalar_legs) step_servo_action<true>(h->P, S, a, nullptr, h->P.friction, any_fn);
    else step_servo_action<false>(h->P, S, a, nullptr, h->P.friction, any_fn);
    S.yaw += a1 * h->P.dt;
    S.yaw_vel = a1;
    gyropod_obs(h->P, S, obs6 + size_t(i) * 6);
    terminated[i] = fabsf(obs6[size_t(i) * 6 + 1]) > h->P.fall_pitch ? 1 : 0;
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

void hostsim_substep(void* hv, int n, float* state, const float* tau) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    substep(h->P, S, tau + size_t(i) * 6, nullptr, h->P.friction, any_fn, NoSync(), nullptr, h->P.joint_limits);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

void hostsim_spine_obs(void* hv, int n, const float* state, float* out) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    spine_observation(h->P, S, out + size_t(i) * UPKIE_SPINE_DIM);
  }
}

// the spine observation as k_spine_obs assembles it: measurement noise on the torques and ImuUncertainty on the IMU
// block, drawn for env tick `tick` (the same draw as the step that produced the state)
void hostsim_spine_obs_with_uncertainty(void* hv, int n, const float* state, uint32_t tick, uint64_t env_offset,
                                        float* out) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    const NoiseCtx nz{env_offset + uint64_t(i), tick};
    float tq[6];
    measured_torques(h->P, S, &nz, tq);
    float* o = out + size_t(i) * UPKIE_SPINE_DIM;
    spine_observation(h->P, S, o, tq);
    apply_imu_uncertainty(h->P, nz, o);
  }
}

void hostsim_sample_init(void* hv, int n, uint64_t seed, uint64_t env_offset, uint64_t episode, float* init) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) sample_init_state(h->P, seed, env_offset + i, episode, init + size_t(i) * UPKIE_INIT_DIM);
}

// one env tick with external forces ext[n][7][3] (same code path as k_step with forces set)
void hostsim_step_servos_ext(void* hv, int n, float* state, const float* action, const float* ext, uint32_t local_mask,
                             float* obs) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    const ExtForces X{ext + size_t(i) * 21, 1, local_mask};
    for (int sub = 0; sub < h->P.nb_substeps; ++sub)
      servo_substep(h->P, S, a, false, nullptr, h->P.friction, any_fn, NoSync(), nullptr, sub, &X, h->P.joint_limits);
    observe_update(h->P, S);
    for (int j = 0; j < 6; ++j) {
      float* o = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = S.torque[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// fp32 controller arithmetic of the kernel, state[n][4] in/out, obs[n][3] = pitch, contact, odometry position
void hostsim_wheel_balancer_step(const UpkieWheelBalancerConfig* c, int n, float* state, const float* obs,
                                 const float* target, float* action) {
  const WheelBalancerParams<float> P{float(c->contact_radius), float(c->dt), float(c->fall_pitch),
                                     float(c->max_ground_velocity), float(c->pitch_damping), float(c->pitch_stiffness),
                                     float(c->position_damping), float(c->position_stiffness),
                                     float(c->stiff_yaw_velocity), float(c->wheel_radius)};
  for (int i = 0; i < n; ++i) {
    WheelBalancerState<float> s{state[4 * i], state[4 * i + 1], state[4 * i + 2], state[4 * i + 3]};
    wheel_balancer_read(P, s, obs[3 * i], obs[3 * i + 2], obs[3 * i + 1] != 0.f, target != nullptr,
                        target ? target[2 * i] : 0.f, target ? target[2 * i + 1] : 0.f);
    wheel_balancer_write(P, s, action + size_t(i) * UPKIE_ACT_DIM, std::nanf(""));
    state[4 * i] = s.ground_velocity; state[4 * i + 1] = s.integral_velocity;
    state[4 * i + 2] = s.target_ground_position; state[4 * i + 3] = s.target_yaw_velocity;
  }
}

void hostsim_gaussian8(uint64_t seed, uint64_t env, uint32_t tick, uint32_t slot, float* out) {
  const NoiseCtx nz{env, tick};
  gaussian8(seed, nz, slot, out);
}

// one env tick with the torque noise models on (same sequence as k_step<.., FAM_EXTRAS, ..>)
void hostsim_step_servos_noise(void* hv, int n, float* state, const float* action, uint32_t tick, uint64_t env_offset,
                               float* obs) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    const NoiseCtx nz{env_offset + uint64_t(i), tick};
    for (int sub = 0; sub < h->P.nb_substeps; ++sub)
      servo_substep(h->P, S, a, false, nullptr, h->P.friction, any_fn, NoSync(), &nz, sub, nullptr, h->P.joint_limits);
    observe_update(h->P, S);
    float tq[6];
    measured_torques(h->P, S, &nz, tq);
    for (int j = 0; j < 6; ++j) {
      float* o = obs + size_t(i) * UPKIE_OBS_DIM + j * 5;
      o[0] = S.q[j]; o[1] = S.qd[j]; o[2] = tq[j]; o[3] = 42.0f; o[4] = 18.0f;
    }
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
  }
}

// spine mode (config.spine_mode): reset = three stopped cycles, step = observation of the first cycle + nb_substeps cycles;
// state[n][STATE_DIM] and lag[n][LAG_DIM] in / out, spine[n][SPINE_DIM] = the assembled observation row
void hostsim_reset_spine(void* hv, int n, float* state, float* lag, const float* init, float* spine) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    SpineLag L;
    reset_robot_spine(h->P, S, L, init + size_t(i) * UPKIE_INIT_DIM, nullptr, h->P.friction, any_fn, h->P.joint_limits);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    lag_to_row(L, lag + size_t(i) * UPKIE_LAG_DIM);
    spine_observation_from_lag(h->P, L, spine + size_t(i) * UPKIE_SPINE_DIM);
  }
}
void hostsim_step_servos_spine(void* hv, int n, float* state, float* lag, const float* action, float* spine) {
  HostSim* h = static_cast<HostSim*>(hv);
  for (int i = 0; i < n; ++i) {
    RobotState S;
    state_from_row(state + size_t(i) * UPKIE_STATE_DIM, S);
    SpineLag L;
    lag_from_row(lag + size_t(i) * UPKIE_LAG_DIM, L);
    float a[UPKIE_ACT_DIM];
    std::memcpy(a, action + size_t(i) * UPKIE_ACT_DIM, sizeof(a));
    clamp_servo_action(h->P, a);
    spine_assemble_observation(S, L);
    for (int sub = 0; sub < h->P.nb_substeps; ++sub)
      spine_cycle(h->P, S, L, a, false, nullptr, h->P.friction, any_fn, NoSync(), h->P.joint_limits);
    state_to_row(S, state + size_t(i) * UPKIE_STATE_DIM);
    lag_to_row(L, lag + size_t(i) * UPKIE_LAG_DIM);
    spine_observation_from_lag(h->P, L, spine + size_t(i) * UPKIE_SPINE_DIM);
  }
}

void hostsim_philox(uint64_t clo, uint64_t chi, uint64_t key, uint32_t* out) {
  Philox4 r = philox4x32_10(clo, chi, key);
  for (int i = 0; i < 4; ++i) out[i] = r.v[i];
}

}  // extern "C"

// ---- MPC core on the host (float = what the kernel runs, double = formulation check) ----
#include <vector>

#include "../../upkie_b200/csrc/mpc_core.cuh"

template <typename T>
static void fill_mpc_params(const UpkieMpcConfig& c, MpcParams<T>& M) {
  const double Ts = c.sampling_period, g = c.gravity;
  const double om = std::sqrt(g / c.leg_length);
  const double ch = std::cosh(Ts * om), sh = std::sinh(Ts * om);
  M.Ts = T(Ts); M.ch = T(ch); M.sho = T(sh / om); M.osh = T(om * sh);
  M.b0 = T(Ts * Ts / 2.0); M.b1 = T(-ch / g + 1.0 / g); M.b2 = T(Ts); M.b3 = T(-om * sh / g);
  M.w_u = T(c.stage_input_cost_weight); M.w_x = T(c.stage_state_cost_weight); M.w_T = T(c.terminal_cost_weight);
  M.a_max = T(c.max_ground_accel); M.v_max = T(c.max_ground_velocity); M.fall_pitch = T(c.fall_pitch);
  M.N = c.nb_timesteps; M.max_iterations = c.max_iterations > 0 ? c.max_iterations : 30;
}

template <typename T>
static void hostsim_mpc_impl(const UpkieMpcConfig* c, int n, const double* x0, const double* v_target,
                             const uint8_t* contact, double dt, double* v_cmd, double* plan, uint8_t* found,
                             int* iterations, uint64_t* active = nullptr, int* work = nullptr) {
  MpcParams<T> M;
  fill_mpc_params(*c, M);
  MpcParams<double> Md;
  fill_mpc_params(*c, Md);
  std::vector<T> tabv(size_t(M.N) * kMpcTabRow);
  mpc_build_tables(Md, tabv.data());
  const T* tab = tabv.data();
  std::vector<T> scratch(size_t(5) * M.N);
  for (int i = 0; i < n; ++i) {
    MpcScratch<T> sc{scratch.data(), 1};
    const T x[4] = {T(x0[4 * i]), T(x0[4 * i + 1]), T(x0[4 * i + 2]), T(x0[4 * i + 3])};
    // `active` ([2][n], in / out): warm start from the previous call's active sets, as k_mpc_step does
    uint64_t up = active ? active[i] : 0, lo = active ? active[size_t(n) + i] : 0;
    T u0 = 0;
    // count iterations by running the solver with increasing caps is wasteful; replicate the loop here
    bool ok = false;
    int it = 0;
    for (; it < M.max_iterations; ++it) {
      if (work) {  // steps of the sweep in the explicit recursion / in the tabulated free tail (cost model)
        const int kmax = mpc_last_bound(up | lo);
        work[2 * i] += kmax + 1;
        work[2 * i + 1] += M.N - 1 - kmax;
      }
      mpc_backward(M, tab, x[0], T(v_target[i]), up, lo, sc);
      uint64_t nu, nl;
      mpc_forward(M, tab, x, up, lo, sc, nu, nl, u0);
      if (nu == up && nl == lo) { ok = true; break; }
      up = nu; lo = nl;
    }
    if (iterations) iterations[i] = it + 1;
    if (active) { active[i] = ok ? up : 0; active[size_t(n) + i] = ok ? lo : 0; }
    for (int k = 0; k < M.N; ++k) {
      double u = double(sc.at(k, 4));
      if (u > c->max_ground_accel) u = c->max_ground_accel;
      if (u < -c->max_ground_accel) u = -c->max_ground_accel;
      plan[size_t(i) * M.N + k] = u;
    }
    found[i] = ok ? 1 : 0;
    v_cmd[i] = double(mpc_command_update(M, T(v_cmd[i]), x[1], contact ? contact[i] != 0 : true, ok, u0, T(dt)));
  }
}

extern "C" {
void hostsim_mpc_step_f32(const UpkieMpcConfig* c, int n, const double* x0, const double* v_target, const uint8_t* contact,
                          double dt, double* v_cmd, double* plan, uint8_t* found, int* iterations) {
  hostsim_mpc_impl<float>(c, n, x0, v_target, contact, dt, v_cmd, plan, found, iterations);
}
void hostsim_mpc_step_f64(const UpkieMpcConfig* c, int n, const double* x0, const double* v_target, const uint8_t* contact,
                          double dt, double* v_cmd, double* plan, uint8_t* found, int* iterations) {
  hostsim_mpc_impl<double>(c, n, x0, v_target, contact, dt, v_cmd, plan, found, iterations);
}
// warm-started form: active[2][n] in / out (the kernel's warm start), work[n][2] += (explicit, tabulated) sweep steps
void hostsim_mpc_step_warm_f32(const UpkieMpcConfig* c, int n, const double* x0, const double* v_target, const uint8_t* contact,
                               double dt, double* v_cmd, double* plan, uint8_t* found, int* iterations, uint64_t* active,
                               int* work) {
  hostsim_mpc_impl<float>(c, n, x0, v_target, contact, dt, v_cmd, plan, found, iterations, active, work);
}
}

// ---- observer pipeline core on the host (fp32, what k_observers_step runs) ----
#include "../../upkie_b200/csrc/observers_core.cuh"

struct HostObservers {
  ObserverParams<float> P;
  std::vector<ObserverState<float>> st;
};

extern "C" {
void* hostsim_observers_create(const UpkieObserverConfig* c, int n) {
  HostObservers* h = new HostObservers();
  h->P.dt = float(c->dt); h->P.cutoff_period = float(c->cutoff_period); h->P.liftoff_inertia = float(c->liftoff_inertia);
  h->P.min_touchdown_acceleration = float(c->min_touchdown_acceleration);
  h->P.min_touchdown_torque = float(c->min_touchdown_torque); h->P.touchdown_inertia = float(c->touchdown_inertia);
  h->P.upper_leg_torque_threshold = float(c->upper_leg_torque_threshold);
  h->P.signed_radius[0] = float(c->signed_radius[0]); h->P.signed_radius[1] = float(c->signed_radius[1]);
  for (int k = 0; k < 9; ++k) h->P.Rbi[k] = float(c->rotation_base_to_imu[k]);
  h->st.assign(size_t(n), ObserverState<float>());
  for (auto& s : h->st) std::memset(&s, 0, sizeof(s));
  return h;
}
void hostsim_observers_destroy(void* h) { delete static_cast<HostObservers*>(h); }
void hostsim_observers_step(void* hv, const float* spine, float* out) {
  HostObservers* h = static_cast<HostObservers*>(hv);
  for (size_t i = 0; i < h->st.size(); ++i)
    observers_step(h->P, h->st[i], spine + i * UPKIE_SPINE_DIM, out + i * UPKIE_OBSV_DIM);
}
}
