"""TEST INFRASTRUCTURE -- CPU restatement of the reference's evaluation bookkeeping (SURVEY 8f-2); never imported by the product.

  EvalOracle.post_step        phc/learning/im_amp.py:244-363 (IMAmpAgent._post_step_eval): termination state, the `curr_max`
                              stopping rule incl. the wrapped last chunk, per-sequence slicing `[:(num_steps - 1)]`, success rate,
                              failed / success keys.
  compute_metrics_lite        smpl_sim.smpllib.smpl_eval.compute_metrics_lite  [3P-memory: smpl_sim is a git dependency
  compute_error_vel / _accel  (requirement.txt:20, unpinned) that is NOT under /root/reference.  Restated from its published
  p_mpjpe                     source: per-frame global / root-relative MPJPE in mm, finite-difference velocity / acceleration
                              errors, Procrustes-aligned MPJPE (the VideoPose3D `p_mpjpe`).]  PARITY UNPINNED for these four:
                              no copy of smpl_sim exists to generate fixtures from.  tests/eval_fp64.py evaluates the same
                              definitions in float64 with a bound on the kernel's fp32 deviation; tests/test_gpu_eval_fp64.py holds
                              the kernel to it frame by frame (frame classes listed there and in DESIGN.md §7), and
                              tests/test_eval_fp64_cpu.py checks that reference, and this fp32 restatement against it.
The bookkeeping half (post_step) follows code that IS under /root/reference and is cited line by line.
"""
from collections import defaultdict

import numpy as np


def compute_error_accel(joints_pred, joints_gt):
    """[T, J, 3] x 2 -> [T - 2]: mean over joints of || (p[t] - 2 p[t+1] + p[t+2])_pred - (...)_gt ||   [3P-memory]"""
    accel_gt = joints_gt[:-2] - 2 * joints_gt[1:-1] + joints_gt[2:]
    accel_pred = joints_pred[:-2] - 2 * joints_pred[1:-1] + joints_pred[2:]
    normed = np.linalg.norm(accel_pred - accel_gt, axis=2)
    return np.mean(normed, axis=1)


def compute_error_vel(joints_pred, joints_gt):
    """[T, J, 3] x 2 -> [T - 1]   [3P-memory]"""
    vel_gt = joints_gt[1:] - joints_gt[:-1]
    vel_pred = joints_pred[1:] - joints_pred[:-1]
    normed = np.linalg.norm(vel_pred - vel_gt, axis=2)
    return np.mean(normed, axis=1)


def p_mpjpe(predicted, target):
    """Procrustes-aligned MPJPE per frame (rigid alignment: rotation, translation, scale), [T, J, 3] x 2 -> [T]   [3P-memory]"""
    assert predicted.shape == target.shape
    muX = np.mean(target, axis=1, keepdims=True)
    muY = np.mean(predicted, axis=1, keepdims=True)
    X0 = target - muX
    Y0 = predicted - muY
    normX = np.sqrt(np.sum(X0 ** 2, axis=(1, 2), keepdims=True))
    normY = np.sqrt(np.sum(Y0 ** 2, axis=(1, 2), keepdims=True))
    X0 = X0 / normX
    Y0 = Y0 / normY
    H = np.matmul(X0.transpose(0, 2, 1), Y0)
    U, s, Vt = np.linalg.svd(H)
    V = Vt.transpose(0, 2, 1)
    R = np.matmul(V, U.transpose(0, 2, 1))
    sign_detR = np.sign(np.expand_dims(np.linalg.det(R), axis=1))
    V[:, :, -1] *= sign_detR
    s[:, -1] *= sign_detR.flatten()
    R = np.matmul(V, U.transpose(0, 2, 1))
    tr = np.expand_dims(np.sum(s, axis=1, keepdims=True), axis=2)
    a = tr * normX / normY
    t = muX - a * np.matmul(muY, R)
    predicted_aligned = a * np.matmul(predicted, R) + t
    return np.mean(np.linalg.norm(predicted_aligned - target, axis=len(target.shape) - 1), axis=len(target.shape) - 2)


def compute_metrics_lite(pred_pos_all, gt_pos_all, root_idx=0, concatenate=True):
    """lists of [T_i, J, 3] -> {'mpjpe_g', 'mpjpe_l', 'mpjpe_pa', 'accel_dist', 'vel_dist'} (mm), per frame, concatenated   [3P-memory]"""
    metrics = defaultdict(list)
    for idx in range(len(pred_pos_all)):
        jpos_gt = gt_pos_all[idx].copy()
        jpos_pred = pred_pos_all[idx].copy()
        mpjpe_g = np.linalg.norm(jpos_gt - jpos_pred, axis=2) * 1000
        vel_dist = compute_error_vel(jpos_pred, jpos_gt) * 1000
        accel_dist = compute_error_accel(jpos_pred, jpos_gt) * 1000
        jpos_pred = jpos_pred - jpos_pred[:, [root_idx]]
        jpos_gt = jpos_gt - jpos_gt[:, [root_idx]]
        pa_mpjpe = p_mpjpe(jpos_pred, jpos_gt) * 1000
        mpjpe = np.linalg.norm(jpos_pred - jpos_gt, axis=2) * 1000
        metrics["mpjpe_g"].append(mpjpe_g)
        metrics["mpjpe_l"].append(mpjpe)
        metrics["mpjpe_pa"].append(pa_mpjpe)
        metrics["accel_dist"].append(accel_dist)
        metrics["vel_dist"].append(vel_dist)
    if concatenate:
        metrics = {k: np.concatenate(v) for k, v in metrics.items()}
    return metrics


class EvalOracle:
    """IMAmpAgent._post_step_eval (im_amp.py:244-363) for a MotionLib stand-in described by:
         num_unique            _motion_lib._num_unique_motions
         keys                  _motion_lib._motion_data_keys (np array of str, one per unique motion)
       per chunk (what load_motions(start_idx=...) leaves behind):
         num_steps [N] int     _motion_lib.get_motion_num_steps()  (motion_lib_base.py:428-432)
         curr_ids  [N] int     _motion_lib._curr_motion_ids
    """

    def __init__(self, num_envs, num_unique, keys):
        self.N, self.num_unique, self.keys = num_envs, num_unique, np.asarray(keys)
        self.terminate_state = np.zeros(num_envs, dtype=bool)          # im_amp.py:143-145
        self.terminate_memory = []
        self.mpjpe, self.mpjpe_all = [], []
        self.gt_pos, self.gt_pos_all = [], []
        self.pred_pos, self.pred_pos_all = [], []
        self.curr_stpes = 0
        self.success_rate = 0
        self.start_idx = 0                                             # humanoid_im.py:439-447

    def post_step(self, terminate, mpjpe, body_pos, body_pos_gt, num_steps, curr_ids):
        """-> (chunk_done, end, info).  terminate [N] bool (info['terminate']), mpjpe [N], body_pos / body_pos_gt [N, J, 3]."""
        end, eval_info = False, {}
        num_steps = np.asarray(num_steps)
        termination_state = np.logical_and(self.curr_stpes <= num_steps - 1, terminate)                   # :249
        self.terminate_state = np.logical_or(termination_state, self.terminate_state)                      # :251
        if (~self.terminate_state).sum() > 0:                                                               # :252
            max_possible_id = self.num_unique - 1
            if (max_possible_id == curr_ids).sum() > 0:                                                     # :255
                bound = int(np.flatnonzero(max_possible_id == curr_ids)[0]) + 1                             # :256
                if (~self.terminate_state[:bound]).sum() > 0:
                    curr_max = num_steps[:bound][~self.terminate_state[:bound]].max()                       # :258-260
                else:
                    curr_max = self.curr_stpes - 1                                                          # :262
            else:
                curr_max = num_steps[~self.terminate_state].max()                                           # :264
            if self.curr_stpes >= curr_max:
                curr_max = self.curr_stpes + 1                                                              # :266
        else:
            curr_max = num_steps.max()                                                                      # :268
        self.mpjpe.append(np.asarray(mpjpe))
        self.gt_pos.append(np.asarray(body_pos_gt))
        self.pred_pos.append(np.asarray(body_pos))
        self.curr_stpes += 1                                                                                # :273
        chunk_done = False
        if self.curr_stpes >= curr_max or self.terminate_state.sum() == self.N:                             # :275
            self.curr_stpes = 0
            self.terminate_memory.append(self.terminate_state.copy())
            self.success_rate = 1 - np.concatenate(self.terminate_memory)[: self.num_unique].mean()         # :278
            all_mpjpe = np.stack(self.mpjpe)
            all_mpjpe = [all_mpjpe[:(i - 1), idx].mean() for idx, i in enumerate(num_steps)]                # :283
            pred = np.stack(self.pred_pos)
            pred = [pred[:(i - 1), idx] for idx, i in enumerate(num_steps)]                                 # :285
            gt = np.stack(self.gt_pos)
            gt = [gt[:(i - 1), idx] for idx, i in enumerate(num_steps)]                                     # :287
            self.mpjpe_all.append(all_mpjpe)
            self.pred_pos_all += pred
            self.gt_pos_all += gt
            if self.start_idx + self.N >= self.num_unique:                                                  # :295
                terminate_hist = np.concatenate(self.terminate_memory)
                succ_idxes = np.flatnonzero(~terminate_hist[: self.num_unique]).tolist()
                pred_succ = [self.pred_pos_all[: self.num_unique][i] for i in succ_idxes]
                gt_succ = [self.gt_pos_all[: self.num_unique][i] for i in succ_idxes]
                pred_all, gt_all = self.pred_pos_all[: self.num_unique], self.gt_pos_all[: self.num_unique]
                failed_keys = self.keys[terminate_hist[: self.num_unique]]
                success_keys = self.keys[~terminate_hist[: self.num_unique]]
                metrics_all = compute_metrics_lite(pred_all, gt_all)
                all_print = {m: np.mean(v) for m, v in metrics_all.items()}
                if len(pred_succ) > 0:
                    metrics_succ = compute_metrics_lite(pred_succ, gt_succ)
                    succ_print = {m: np.mean(v) for m, v in metrics_succ.items()}
                else:
                    succ_print = all_print                                                                  # :322-324 ("No success!!!")
                end = True
                eval_info = {"eval_success_rate": self.success_rate, "eval_mpjpe_all": all_print["mpjpe_g"],   # :333-342
                             "eval_mpjpe_succ": succ_print["mpjpe_g"], "accel_dist": succ_print["accel_dist"],
                             "vel_dist": succ_print["vel_dist"], "mpjpel_all": all_print["mpjpe_l"],
                             "mpjpel_succ": succ_print["mpjpe_l"], "mpjpe_pa": succ_print["mpjpe_pa"]}
                return True, True, {"end": end, "eval_info": eval_info, "failed_keys": failed_keys, "success_keys": success_keys}
            chunk_done = True                                                                               # :351 done[:] = 1
            self.start_idx += self.N                                                                        # :353 forward_motion_samples
            self.terminate_state = np.zeros(self.N, dtype=bool)
            self.mpjpe, self.gt_pos, self.pred_pos = [], [], []
        return chunk_done, end, {"end": end, "eval_info": eval_info, "failed_keys": [], "success_keys": []}
