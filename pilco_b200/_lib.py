"""ctypes binding of ``libpilco_b200.so`` (the C ABI declared in ``include/pilco_b200.h``).

The product path has no CPU fallback: if the shared library is missing the import of this module
raises, and every compute entry point raises unless a CUDA device is present.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PILCO_B200_LIB") or os.path.join(_HERE, "libpilco_b200.so")   # env: diagnostics builds

c_dp = C.c_void_p          # device pointers are passed as integers (tensor.data_ptr())
c_ll = C.c_longlong


class GpModel(C.Structure):
    """mirror of ``pilco_gp_model``"""
    _fields_ = [("n", C.c_int), ("D", C.c_int), ("E", C.c_int), ("mode", C.c_int),
                ("X", c_dp), ("X_bs", c_ll),
                ("ell", c_dp), ("ell_bs", c_ll),
                ("sf2", c_dp), ("sf2_bs", c_ll),
                ("beta", c_dp), ("beta_bs", c_ll),
                ("iK", c_dp), ("ldk", C.c_int)]


class Policy(C.Structure):
    """mirror of ``pilco_policy``"""
    _fields_ = [("kind", C.c_int), ("Ds", C.c_int), ("U", C.c_int), ("squash", C.c_int),
                ("max_action", c_dp),
                ("W", c_dp), ("W_bs", c_ll), ("b", c_dp), ("b_bs", c_ll),
                ("rbf", GpModel)]


class RewardTerm(C.Structure):
    """mirror of ``pilco_reward_term``"""
    _fields_ = [("kind", C.c_int), ("channel", C.c_int), ("coef", C.c_double), ("W", c_dp), ("t", c_dp)]


class Rollout(C.Structure):
    """mirror of ``pilco_rollout``"""
    _fields_ = [("R", C.c_int), ("H", C.c_int),
                ("dyn", GpModel), ("pol", Policy),
                ("n_rewards", C.c_int), ("rewards", RewardTerm * 8),
                ("m0", c_dp), ("m0_bs", c_ll), ("S0", c_dp), ("S0_bs", c_ll),
                ("traj_m", c_dp), ("traj_S", c_dp), ("reward", c_dp), ("step_reward", c_dp),
                ("info", c_dp), ("ws", c_dp), ("ws_bytes", C.c_size_t),
                ("mult_mu", C.c_double), ("step_risk", c_dp),
                ("tape", c_dp), ("tape_bytes", C.c_size_t)]


class RolloutGrad(C.Structure):
    """mirror of ``pilco_rollout_grad``"""
    _fields_ = [("gW", c_dp), ("gb", c_dp), ("gXc", c_dp), ("gYc", c_dp), ("gell", c_dp), ("pol_L", c_dp),
                ("gm0", c_dp), ("gS0", c_dp), ("ws", c_dp), ("ws_bytes", C.c_size_t)]


class Particles(C.Structure):
    """mirror of ``pilco_particles``"""
    _fields_ = [("P", C.c_int), ("H", C.c_int),
                ("dyn", GpModel), ("pol", Policy),
                ("n_rewards", C.c_int), ("rewards", RewardTerm * 8), ("mult_mu", C.c_double),
                ("x0", c_dp), ("eps", c_dp),
                ("traj", c_dp), ("act", c_dp), ("step_reward", c_dp), ("step_risk", c_dp), ("ret", c_dp),
                ("ws", c_dp), ("ws_bytes", C.c_size_t)]


class ParticlesGrad(C.Structure):
    """mirror of ``pilco_particles_grad``"""
    _fields_ = [("gW", c_dp), ("gb", c_dp), ("gXc", c_dp), ("gYc", c_dp), ("gell", c_dp), ("pol_L", c_dp),
                ("value", c_dp), ("ws", c_dp), ("ws_bytes", C.c_size_t)]


class Angles(C.Structure):
    """mirror of ``pilco_angles``"""
    _fields_ = [("A", C.c_int), ("dims", C.c_int * 16)]


class Exploration(C.Structure):
    """mirror of ``pilco_exploration``"""
    _fields_ = [("b", C.c_double), ("step_var", c_dp)]


class ObsNoise(C.Structure):
    """mirror of ``pilco_obs_noise``"""
    _fields_ = [("var", C.c_double * 16)]


class ParticlesNoise(C.Structure):
    """mirror of ``pilco_particles_noise``"""
    _fields_ = [("v", ObsNoise), ("nu", c_dp)]


class PolicySchedule(C.Structure):
    """mirror of ``pilco_policy_schedule``"""
    _fields_ = [("W_ts", c_ll), ("b_ts", c_ll)]


class ParticlesResample(C.Structure):
    """mirror of ``pilco_particles_resample``"""
    _fields_ = [("xi", c_dp), ("step_mean", c_dp), ("step_cov", c_dp)]


class Mlp(C.Structure):
    """mirror of ``pilco_mlp``"""
    _fields_ = [("L", C.c_int), ("width", C.c_int * 2), ("theta", c_dp), ("theta_bs", c_ll), ("gtheta", c_dp)]


class FeatureDraws(C.Structure):
    """mirror of ``pilco_feature_draws``"""
    _fields_ = [("F", C.c_int), ("omega", c_dp), ("w", c_dp), ("v", c_dp)]


class Cem(C.Structure):
    """mirror of ``pilco_cem``"""
    _fields_ = [("K", C.c_int), ("H", C.c_int), ("U", C.c_int), ("n_elite", C.c_int),
                ("alpha", C.c_double), ("lo", C.c_double), ("hi", C.c_double),
                ("value", c_dp), ("cand", c_dp), ("xi", c_dp), ("mean", c_dp), ("std", c_dp),
                ("best_value", c_dp), ("best", c_dp), ("trace", c_dp)]


class Adam(C.Structure):
    """mirror of ``pilco_adam``"""
    _fields_ = [("R", C.c_int), ("n", C.c_int), ("lr", C.c_double), ("b1", C.c_double), ("b2", C.c_double),
                ("eps", C.c_double), ("max_norm", C.c_double), ("theta", c_dp), ("ld_theta", C.c_int),
                ("packed", c_dp), ("ld_packed", C.c_int), ("m", c_dp), ("v", c_dp), ("t", c_dp), ("b1t", c_dp),
                ("b2t", c_dp), ("iter", c_dp), ("trace", c_dp), ("ok", c_dp), ("trace_rows", C.c_int)]


MAX_FEATURES = 8192                              # PILCO_MAX_FEATURES
CEM_MAX_K = 8192                                 # pilco_cem_update's largest K
POLICY_LINEAR, POLICY_RBF, POLICY_MLP = 0, 1, 2
REWARD_EXP, REWARD_LINEAR, REWARD_BOX = 0, 1, 2
REWARD_EXP_SA, REWARD_LINEAR_SA = 3, 4           # on the joint state-action Gaussian [x, u], D = Ds + U
JOINT_REWARDS = (REWARD_EXP_SA, REWARD_LINEAR_SA)
CHANNEL_ADD, CHANNEL_MULT = 0, 1
ABI_VERSION = 3
ABI_MAX_D = 16                                   # PILCO_MAX_D

_PAN = [C.POINTER(Particles), C.POINTER(Angles), C.POINTER(ParticlesNoise)]     # the noisy particle calls' first three

_RAEN = [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(Exploration), C.POINTER(ObsNoise)]   # the noisy rollout's

# name -> (restype, argtypes); every symbol declared in include/pilco_b200.h
SIGNATURES = {
    "pilco_version": (C.c_int, []),
    "pilco_status_string": (C.c_char_p, [C.c_int]),
    "pilco_pad_n": (C.c_int, [C.c_int]),
    "pilco_mm_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "pilco_mm_forward": (C.c_int, [C.POINTER(GpModel), C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                   c_dp, C.c_size_t, c_dp]),
    "pilco_gp_factorize_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "pilco_gp_factorize": (C.c_int, [C.c_int] * 4 + [c_dp, c_ll] * 5 + [c_dp, C.c_int, c_dp, c_dp,
                                                                        c_dp, C.c_size_t, c_dp]),
    "pilco_gp_append_tri_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "pilco_gp_append_tri": (C.c_int, [C.c_int] * 4 + [c_dp] * 5 + [c_dp, C.c_int] * 4 + [c_dp, c_dp,
                                                                              c_dp, C.c_size_t, c_dp]),
    "pilco_gp_nlml_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "pilco_gp_nlml": (C.c_int, [C.c_int] * 4 + [c_dp, c_ll] * 5 + [c_dp] * 5 + [c_dp, C.c_size_t, c_dp]),
    "pilco_fitc_nlml_workspace_bytes": (C.c_size_t, [C.c_int] * 5),
    "pilco_fitc_nlml": (C.c_int, [C.c_int] * 5 + [c_dp] * 6 + [c_dp] * 6 + [c_dp, C.c_size_t, c_dp]),
    "pilco_fitc_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "pilco_fitc_factorize": (C.c_int, [C.c_int] * 4 + [c_dp] * 6 + [c_dp, C.c_int, c_dp, c_dp, c_dp,
                                                                  C.c_size_t, c_dp]),
    "pilco_gp_predict_workspace_bytes": (C.c_size_t, [C.c_int] * 5),
    "pilco_gp_predict": (C.c_int, [C.POINTER(GpModel), C.c_int, C.c_int, C.c_int, c_dp, c_dp, c_dp, C.c_int,
                                   c_dp, C.c_size_t, c_dp]),
    "pilco_gp_predict_samples_workspace_bytes": (C.c_size_t, [C.c_int] * 6),
    "pilco_gp_predict_samples": (C.c_int, [C.POINTER(GpModel)] + [C.c_int] * 4 + [c_dp] * 3 + [C.c_int, C.c_double, c_dp,
                                                                                             c_dp, C.c_size_t, c_dp]),
    "pilco_squash_sin": (C.c_int, [C.c_int, C.c_int] + [c_dp] * 7),
    "pilco_linear_action": (C.c_int, [C.c_int] * 3 + [c_dp, c_ll, c_dp, c_ll] + [c_dp] * 6),
    "pilco_exp_reward": (C.c_int, [C.c_int, C.c_int] + [c_dp] * 8),
    "pilco_box_risk": (C.c_int, [C.c_int, C.c_int] + [c_dp] * 7),
    "pilco_rollout_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout)]),
    "pilco_rollout_tape_bytes": (C.c_size_t, [C.POINTER(Rollout)]),
    "pilco_mm_tape_bytes": (C.c_size_t, [C.c_int] * 4),
    "pilco_mm_tape_bwd_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "pilco_mm_forward_taped": (C.c_int, [C.POINTER(GpModel), C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                         c_dp, C.c_size_t, c_dp, C.c_size_t, c_dp]),
    "pilco_mm_backward_taped": (C.c_int, [C.POINTER(GpModel), C.c_int] + [c_dp] * 6 + [c_dp, C.c_size_t, c_dp, c_dp,
                                                                                  c_dp, C.c_size_t, c_dp]),
    "pilco_rollout_forward": (C.c_int, [C.POINTER(Rollout), c_dp]),
    "pilco_mm_bwd_workspace_bytes": (C.c_size_t, [C.c_int] * 5),
    "pilco_mm_backward": (C.c_int, [C.POINTER(GpModel), C.c_int] + [c_dp] * 11 + [c_dp, C.c_size_t, c_dp]),
    "pilco_rollout_bwd_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout)]),
    "pilco_rollout_backward": (C.c_int, [C.POINTER(Rollout), C.POINTER(RolloutGrad), c_dp]),
    "pilco_trig_moments": (C.c_int, [C.c_int, C.c_int, C.POINTER(Angles)] + [c_dp] * 6),
    "pilco_rollout_angles_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles)]),
    "pilco_rollout_angles_tape_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles)]),
    "pilco_rollout_angles_bwd_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles)]),
    "pilco_rollout_angles_forward": (C.c_int, [C.POINTER(Rollout), C.POINTER(Angles), c_dp]),
    "pilco_rollout_angles_backward": (C.c_int, [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(RolloutGrad), c_dp]),
    "pilco_rollout_explore_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles),
                                                           C.POINTER(Exploration)]),
    "pilco_rollout_explore_bwd_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles),
                                                               C.POINTER(Exploration)]),
    "pilco_rollout_explore_forward": (C.c_int, [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(Exploration), c_dp]),
    "pilco_rollout_explore_backward": (C.c_int, [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(Exploration),
                                                 C.POINTER(RolloutGrad), c_dp]),
    "pilco_rollout_noisy_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(Exploration),
                                                         C.POINTER(ObsNoise)]),
    "pilco_rollout_noisy_bwd_workspace_bytes": (C.c_size_t, [C.POINTER(Rollout), C.POINTER(Angles),
                                                             C.POINTER(Exploration), C.POINTER(ObsNoise)]),
    "pilco_rollout_noisy_forward": (C.c_int, [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(Exploration),
                                              C.POINTER(ObsNoise), c_dp]),
    "pilco_rollout_noisy_backward": (C.c_int, [C.POINTER(Rollout), C.POINTER(Angles), C.POINTER(Exploration),
                                               C.POINTER(ObsNoise), C.POINTER(RolloutGrad), c_dp]),
    "pilco_rollout_scheduled_workspace_bytes": (C.c_size_t, _RAEN + [C.POINTER(PolicySchedule)]),
    "pilco_rollout_scheduled_forward": (C.c_int, _RAEN + [C.POINTER(PolicySchedule), c_dp]),
    "pilco_rollout_scheduled_bwd_workspace_bytes": (C.c_size_t, _RAEN + [C.POINTER(PolicySchedule)]),
    "pilco_rollout_scheduled_backward": (C.c_int, _RAEN + [C.POINTER(PolicySchedule), C.POINTER(RolloutGrad), c_dp]),
    "pilco_particles_workspace_bytes": (C.c_size_t, [C.POINTER(Particles)]),
    "pilco_particles_rollout": (C.c_int, [C.POINTER(Particles), c_dp]),
    "pilco_gp_predict_vjp_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "pilco_gp_predict_vjp": (C.c_int, [C.POINTER(GpModel), C.c_int] + [c_dp] * 5 + [C.c_size_t, c_dp]),
    "pilco_particles_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles)]),
    "pilco_particles_rollout_grad": (C.c_int, [C.POINTER(Particles), C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_batch_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.c_int]),
    "pilco_particles_rollout_batch_grad": (C.c_int, [C.POINTER(Particles), C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_consistent_workspace_bytes": (C.c_size_t, [C.POINTER(Particles)]),
    "pilco_particles_rollout_consistent": (C.c_int, [C.POINTER(Particles), c_dp]),
    "pilco_particles_consistent_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.c_int]),
    "pilco_particles_rollout_consistent_grad": (C.c_int, [C.POINTER(Particles), C.c_int, C.POINTER(ParticlesGrad),
                                                          c_dp]),
    "pilco_particles_score_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.c_int]),
    "pilco_particles_rollout_score_grad": (C.c_int, [C.POINTER(Particles), C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_angles_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Angles)]),
    "pilco_particles_angles_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Angles), c_dp]),
    "pilco_particles_angles_consistent_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Angles)]),
    "pilco_particles_angles_consistent_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Angles), c_dp]),
    "pilco_particles_angles_batch_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Angles),
                                                                       C.c_int]),
    "pilco_particles_angles_batch_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Angles), C.c_int,
                                                            C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_angles_consistent_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Angles),
                                                                            C.c_int]),
    "pilco_particles_angles_consistent_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Angles), C.c_int,
                                                                 C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_angles_score_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Angles),
                                                                       C.c_int]),
    "pilco_particles_angles_score_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Angles), C.c_int,
                                                            C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_noisy_workspace_bytes": (C.c_size_t, _PAN),
    "pilco_particles_noisy_rollout": (C.c_int, _PAN + [c_dp]),
    "pilco_particles_noisy_consistent_workspace_bytes": (C.c_size_t, _PAN),
    "pilco_particles_noisy_consistent_rollout": (C.c_int, _PAN + [c_dp]),
    "pilco_particles_noisy_batch_grad_workspace_bytes": (C.c_size_t, _PAN + [C.c_int]),
    "pilco_particles_noisy_batch_grad_rollout": (C.c_int, _PAN + [C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_noisy_consistent_grad_workspace_bytes": (C.c_size_t, _PAN + [C.c_int]),
    "pilco_particles_noisy_consistent_grad_rollout": (C.c_int, _PAN + [C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_noisy_score_grad_workspace_bytes": (C.c_size_t, _PAN + [C.c_int]),
    "pilco_particles_noisy_score_grad_rollout": (C.c_int, _PAN + [C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_explore_batch_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(Exploration), C.c_int]),
    "pilco_particles_explore_batch_grad_rollout": (C.c_int, _PAN + [C.POINTER(Exploration), C.c_int,
                                                                    C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_explore_consistent_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(Exploration), C.c_int]),
    "pilco_particles_explore_consistent_grad_rollout": (C.c_int, _PAN + [C.POINTER(Exploration), C.c_int,
                                                                         C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_consistent_score_grad_workspace_bytes": (C.c_size_t, _PAN + [C.c_int]),
    "pilco_particles_consistent_score_grad_rollout": (C.c_int, _PAN + [C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_resampled_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(ParticlesResample)]),
    "pilco_particles_resampled_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(ParticlesResample), c_dp]),
    "pilco_particles_resampled_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(ParticlesResample),
                                                                    C.c_int]),
    "pilco_particles_resampled_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(ParticlesResample), C.c_int,
                                                         C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_scheduled_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(PolicySchedule)]),
    "pilco_particles_scheduled_rollout": (C.c_int, _PAN + [C.POINTER(PolicySchedule), c_dp]),
    "pilco_particles_scheduled_consistent_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(PolicySchedule)]),
    "pilco_particles_scheduled_consistent_rollout": (C.c_int, _PAN + [C.POINTER(PolicySchedule), c_dp]),
    "pilco_particles_scheduled_batch_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(Exploration),
                                                                                 C.POINTER(PolicySchedule), C.c_int]),
    "pilco_particles_scheduled_batch_grad_rollout": (C.c_int, _PAN + [C.POINTER(Exploration), C.POINTER(PolicySchedule),
                                                                      C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_scheduled_consistent_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(Exploration),
                                                                                      C.POINTER(PolicySchedule),
                                                                                      C.c_int]),
    "pilco_particles_scheduled_consistent_grad_rollout": (C.c_int, _PAN + [C.POINTER(Exploration),
                                                                           C.POINTER(PolicySchedule), C.c_int,
                                                                           C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_scheduled_score_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(PolicySchedule), C.c_int]),
    "pilco_particles_scheduled_score_grad_rollout": (C.c_int, _PAN + [C.POINTER(PolicySchedule), C.c_int,
                                                                      C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_scheduled_consistent_score_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(PolicySchedule),
                                                                                            C.c_int]),
    "pilco_particles_scheduled_consistent_score_grad_rollout": (C.c_int, _PAN + [C.POINTER(PolicySchedule), C.c_int,
                                                                                 C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_scheduled_resampled_workspace_bytes": (C.c_size_t, [C.POINTER(Particles),
                                                                         C.POINTER(ParticlesResample),
                                                                         C.POINTER(PolicySchedule)]),
    "pilco_particles_scheduled_resampled_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(ParticlesResample),
                                                              C.POINTER(PolicySchedule), c_dp]),
    "pilco_particles_scheduled_resampled_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles),
                                                                              C.POINTER(ParticlesResample),
                                                                              C.POINTER(PolicySchedule), C.c_int]),
    "pilco_particles_scheduled_resampled_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(ParticlesResample),
                                                                   C.POINTER(PolicySchedule), C.c_int,
                                                                   C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_mlp_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp)]),
    "pilco_particles_mlp_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp), c_dp]),
    "pilco_particles_mlp_consistent_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp)]),
    "pilco_particles_mlp_consistent_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp), c_dp]),
    "pilco_particles_mlp_resampled_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                   C.POINTER(ParticlesResample)]),
    "pilco_particles_mlp_resampled_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp),
                                                        C.POINTER(ParticlesResample), c_dp]),
    "pilco_particles_mlp_batch_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                    C.POINTER(Exploration), C.c_int]),
    "pilco_particles_mlp_batch_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp), C.POINTER(Exploration),
                                                         C.c_int, C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_mlp_consistent_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                         C.POINTER(Exploration), C.c_int]),
    "pilco_particles_mlp_consistent_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp),
                                                              C.POINTER(Exploration), C.c_int,
                                                              C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_mlp_resampled_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                        C.POINTER(ParticlesResample), C.c_int]),
    "pilco_particles_mlp_resampled_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp),
                                                             C.POINTER(ParticlesResample), C.c_int,
                                                             C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_features_draw_workspace_bytes": (C.c_size_t, [C.POINTER(GpModel), C.c_int, C.c_int]),
    "pilco_particles_features_draw": (C.c_int, [C.POINTER(GpModel), c_dp, C.c_int, C.c_int] + [c_dp] * 6
                                      + [C.c_size_t, c_dp]),
    "pilco_particles_features_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(FeatureDraws)]),
    "pilco_particles_features_rollout": (C.c_int, _PAN + [C.POINTER(FeatureDraws), c_dp]),
    "pilco_particles_features_grad_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(Exploration),
                                                                          C.POINTER(FeatureDraws), C.c_int]),
    "pilco_particles_features_grad_rollout": (C.c_int, _PAN + [C.POINTER(Exploration), C.POINTER(FeatureDraws), C.c_int,
                                                               C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_mlp_features_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                  C.POINTER(FeatureDraws)]),
    "pilco_particles_mlp_features_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp), C.POINTER(FeatureDraws),
                                                       c_dp]),
    "pilco_particles_mlp_features_grad_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                       C.POINTER(Exploration), C.POINTER(FeatureDraws),
                                                                       C.c_int]),
    "pilco_particles_mlp_features_grad_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp),
                                                            C.POINTER(Exploration), C.POINTER(FeatureDraws), C.c_int,
                                                            C.POINTER(ParticlesGrad), c_dp]),
    "pilco_particles_scheduled_batch_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(PolicySchedule), C.c_int]),
    "pilco_particles_scheduled_batch_rollout": (C.c_int, _PAN + [C.POINTER(PolicySchedule), C.c_int, c_dp, c_dp]),
    "pilco_particles_scheduled_consistent_batch_workspace_bytes": (C.c_size_t, _PAN + [C.POINTER(PolicySchedule),
                                                                                       C.c_int]),
    "pilco_particles_scheduled_consistent_batch_rollout": (C.c_int, _PAN + [C.POINTER(PolicySchedule), C.c_int, c_dp,
                                                                            c_dp]),
    "pilco_particles_batch_workspace_bytes": (C.c_size_t, _PAN + [C.c_int]),
    "pilco_particles_batch_rollout": (C.c_int, _PAN + [C.c_int, c_dp, c_dp]),
    "pilco_particles_consistent_batch_workspace_bytes": (C.c_size_t, _PAN + [C.c_int]),
    "pilco_particles_consistent_batch_rollout": (C.c_int, _PAN + [C.c_int, c_dp, c_dp]),
    "pilco_particles_mlp_batch_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp), C.c_int]),
    "pilco_particles_mlp_batch_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp), C.c_int, c_dp, c_dp]),
    "pilco_particles_mlp_consistent_batch_workspace_bytes": (C.c_size_t, [C.POINTER(Particles), C.POINTER(Mlp),
                                                                          C.c_int]),
    "pilco_particles_mlp_consistent_batch_rollout": (C.c_int, [C.POINTER(Particles), C.POINTER(Mlp), C.c_int, c_dp,
                                                               c_dp]),
    "pilco_cem_update_workspace_bytes": (C.c_size_t, [C.c_int]),
    "pilco_cem_update": (C.c_int, [C.POINTER(Cem), c_dp, C.c_size_t, c_dp]),
    "pilco_cem_draw": (C.c_int, [C.POINTER(Cem), c_dp]),
    "pilco_normals": (C.c_int, [C.c_ulonglong, C.c_uint, c_dp, c_ll, c_dp, c_dp]),
    "pilco_adam_update": (C.c_int, [C.POINTER(Adam), c_dp]),
    "pilco_particles_reward_moments": (C.c_int, [C.POINTER(Particles), C.POINTER(Angles), C.c_int, c_dp, c_dp, c_dp]),
    "pilco_mm_forward_profile": (C.c_int, [C.POINTER(GpModel), C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                           c_dp, C.c_size_t, C.POINTER(C.c_float), c_dp]),
    "pilco_mm_forward_taped_profile": (C.c_int, [C.POINTER(GpModel), C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                                 c_dp, C.c_size_t, c_dp, C.c_size_t, C.POINTER(C.c_float), c_dp]),
    "pilco_microbench_fp64": (C.c_int, [C.c_int, C.c_int, C.c_int, c_dp, C.POINTER(C.c_float), c_dp]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "pilco_b200: %s is missing -- build it with `python -m pilco_b200.build` "
            "(there is no CPU fallback for the moment-matching path)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export the symbol
        fn.restype = res
        fn.argtypes = args
    if lib.pilco_version() != ABI_VERSION:
        raise RuntimeError("pilco_b200: ABI version mismatch")
    return lib


lib = _load()


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("pilco_b200 %s failed: %s (status %d)" %
                           (what, lib.pilco_status_string(rc).decode(), rc))
