"""TEST INFRASTRUCTURE: a stand-in for mcl_3dl_b200.engine whose Engine runs on the HOST through tests/hostsim (the
product's per-thread device functions compiled for the host).  It lets the CPU suite execute the bodies of GPU tests
whose kernels are thin wrappers around those functions (tests/test_gpu_resident.py), so that a failure on the H100 can
only come from the kernels / plumbing, not from the tests' own expectations.  Never imported by the product."""
import ctypes as C
import os

import numpy as np

from mcl_3dl_b200 import engine as real
from mcl_3dl_b200 import synth

HS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
LikParams = real.LikParams
beam_params_from_reference = real.beam_params_from_reference


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else None


class Engine:
    def __init__(self, devices=(0,), lib_path=None):
        L = C.CDLL(os.path.join(HS, "libhostsim.so"))
        vp, sz = C.c_void_p, C.c_size_t
        L.hostsim_measure.argtypes = [vp, sz, vp, vp, C.c_float, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp]
        L.hostsim_pf_predict.argtypes = [vp, vp, C.c_float, C.c_float, C.c_float, vp, sz]
        L.hostsim_pf_resample_philox.argtypes = [vp, vp, sz, C.c_float, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp, vp, vp]
        L.hostsim_pf_estimate.argtypes = [vp, vp, sz, vp, C.c_float, C.c_float, vp, vp, vp, vp, vp]
        self.L = L
        self.calls = 0

    def close(self):
        pass

    def set_map(self, map_pts, lik=None, beam=None, stamp=1):
        self.map, self.lik, self.beam = np.ascontiguousarray(map_pts, dtype=synth.POINT), lik, beam

    def _records(self, poses, lik_pts, beam_pts, origins):
        poses = np.ascontiguousarray(poses, dtype=synth.POSE)
        lik_pts = np.ascontiguousarray(lik_pts if lik_pts is not None else np.zeros(0, synth.POINT), dtype=synth.POINT)
        beam_pts = np.ascontiguousarray(beam_pts if beam_pts is not None else np.zeros(0, synth.POINT), dtype=synth.POINT)
        origins = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(poses), dtype=synth.RESULT)
        rc = self.L.hostsim_measure(_ptr(self.map), len(self.map), C.byref(self.lik) if self.lik is not None else None,
                                    C.byref(self.beam) if self.beam is not None else None, 1.0, _ptr(poses), len(poses),
                                    _ptr(lik_pts), len(lik_pts), _ptr(beam_pts), len(beam_pts), _ptr(origins), len(origins),
                                    _ptr(out), None)
        assert rc == 0
        return out, len(lik_pts)

    @staticmethod
    def _update(rec, n_lik, prior, extra):
        """weight_kernel / normalize_kernel restated with numpy (float32 products, float64 sums as on the device)."""
        lk = (np.float32(1.0) * rec["score_beam"]).astype(np.float32)
        lk = (lk * rec["score_like"]).astype(np.float32)
        if extra is not None:
            lk = (lk * extra).astype(np.float32)
        w = (prior * lk).astype(np.float32)
        total = np.float32(w.astype(np.float64).sum())
        q = rec["match_cnt"].astype(np.float32) / np.float32(n_lik) if n_lik else np.zeros(len(w), np.float32)
        summ = {"weight_sum": float(total), "kept": int(total > 0), "match_ratio_min": float(min(np.float32(1.0), q.min())),
                "match_ratio_max": float(max(np.float32(0.0), q.max())), "entropy": 0.0, "max_index": 0}
        if total > 0:
            post = (w / total).astype(np.float32)
            nz = post > 0
            summ["entropy"] = float(np.float32(-(post[nz] * np.log(post[nz]).astype(np.float32)).astype(np.float64).sum()))
            summ["max_index"] = int(np.argmax(post))
        else:
            post = prior.copy()
        return post, summ

    def measure_update(self, poses, lik_pts, beam_pts, origins, prior, extra_likelihood=None, want_records=False):
        rec, n_lik = self._records(poses, lik_pts, beam_pts, origins)
        prior = np.ascontiguousarray(prior, dtype=np.float32)
        extra = np.ascontiguousarray(extra_likelihood, dtype=np.float32) if extra_likelihood is not None else None
        post, summ = self._update(rec, n_lik, prior, extra)
        return post, summ, rec if want_records else None

    # ---- resident particle set
    def particles_set(self, states, prob):
        self.states = np.array(states, dtype=synth.STATE)
        self.prob = np.array(prob, dtype=np.float32)

    def particles_get(self):
        return self.states.copy(), self.prob.copy()

    def particles_predict(self, odom_prev, odom_current, time_diff, tc_lin, tc_ang):
        a = np.ascontiguousarray(odom_prev, dtype=synth.POSE).reshape(1)
        b = np.ascontiguousarray(odom_current, dtype=synth.POSE).reshape(1)
        assert self.L.hostsim_pf_predict(_ptr(a), _ptr(b), time_diff, tc_lin, tc_ang, _ptr(self.states), len(self.states)) == 0

    def particles_measure_update(self, lik_pts, beam_pts, origins, odom_err_integ_lin_sigma=0.0):
        poses = synth.make_poses(self.states["pos"], self.states["rot"])   # pf_pack_kernel
        extra = None
        if odom_err_integ_lin_sigma > 0:
            s = float(np.float32(odom_err_integ_lin_sigma))
            a, sq2 = np.float32(1.0 / np.sqrt(2.0 * np.pi * s * s)), np.float32(s * s * 2.0)
            lin = self.states["odom_err_integ_lin"]
            x = np.sqrt((lin[:, 0] * lin[:, 0] + lin[:, 1] * lin[:, 1]).astype(np.float32) + lin[:, 2] * lin[:, 2]).astype(np.float32)
            extra = (a * np.exp((-x * x / sq2).astype(np.float32)).astype(np.float32)).astype(np.float32)
        rec, n_lik = self._records(poses, lik_pts, beam_pts, origins)
        self.prob, summ = self._update(rec, n_lik, self.prob, extra)
        return summ

    def particles_resample(self, sigma_pos, sigma_rpy, initial_frac, seed):
        n = len(self.states)
        sp = np.ascontiguousarray(sigma_pos, dtype=np.float32)
        sr = np.ascontiguousarray(sigma_rpy, dtype=np.float32)
        out = np.zeros(n, dtype=synth.STATE)
        out_p = np.zeros(n, dtype=np.float32)
        self.calls += 1
        assert self.L.hostsim_pf_resample_philox(_ptr(self.prob), _ptr(self.states), n, initial_frac, seed, self.calls, _ptr(sp),
                                                 _ptr(sr), _ptr(out), _ptr(out_p), None, None, None) == 0
        self.states, self.prob = out, out_p

    def particles_estimate(self, state_prev=None, bias_var_dist=1.0, bias_var_ang=1.0):
        prev = np.ascontiguousarray(state_prev, dtype=synth.POSE).reshape(1) if state_prev is not None else None
        pos, rot, cov = np.zeros(3, np.float32), np.zeros(4, np.float32), np.zeros(36, np.float32)
        best, wsum = C.c_uint32(0), C.c_float(0)
        assert self.L.hostsim_pf_estimate(_ptr(self.prob), _ptr(self.states), len(self.states), _ptr(prev) if prev is not None else None,
                                          bias_var_dist, bias_var_ang, _ptr(pos), _ptr(rot), C.byref(best), C.byref(wsum), _ptr(cov)) == 0
        i = int(best.value)
        return {"mean_biased": synth.make_poses([pos], [rot]), "max_state": synth.make_poses([self.states["pos"][i]], [self.states["rot"][i]]),
                "max_index": i, "weight_sum_biased": float(wsum.value), "cov": cov.reshape(6, 6)}
