"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / initcheck / synccheck), covering every kernel the
library ships: map build incl. the NN field, the likelihood kernels with and without the NN field + the field mode, both
beam kernels x both raycasters, the fused weight update, the resident particle set (predict / update / estimate /
resample), the scan preprocessing and the normal-weighted sampler.
   compute-sanitizer --tool racecheck python profiles/sanitize.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcl_3dl_b200 import engine, synth  # noqa: E402

s = synth.scene(20_000, 70, 96, 40, seed=3)
for env in ({}, {"MCL3DL_NNF": "0"}, {"MCL3DL_BEAM": "dq"}, {"MCL3DL_BEAM": "pl"}):
    for k in ("MCL3DL_NNF", "MCL3DL_BEAM"):
        os.environ.pop(k, None)
    os.environ.update(env)
    for use_dda in (True, False):
        eng = engine.Engine((0,))
        lik = engine.LikParams(dist_weight=(1, 1, 5))
        beam = engine.beam_params_from_reference(num_points_default=40, use_raycast_using_dda=use_dda)
        eng.set_map(s["map"], lik, beam)
        r = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
        st = eng.beam_status(s["particles"][:5], s["beam"], s["origins"])
        print(env, "dda" if use_dda else "kd", int(r["match_cnt"].sum()), int(r["n_hit"].sum()), st.shape)
        eng.close()
for k in ("MCL3DL_NNF", "MCL3DL_BEAM"):
    os.environ.pop(k, None)
eng = engine.Engine((0,))
eng.set_map(s["map"], engine.LikParams(dist_weight=(1, 1, 5)), engine.beam_params_from_reference(num_points_default=40))
prior = np.full(70, 1.0 / 70, np.float32)
post, summ, rec = eng.measure_update(s["particles"], s["lik"], s["beam"], s["origins"], prior, want_records=True)
print("fused update", summ["kept"], round(summ["entropy"], 3))
eng.field_mode(True)
f = eng.measure(s["particles"], s["lik"], None, None)
eng.field_mode(False)
print("field mode", int(f["match_cnt"].sum()))
st = np.zeros(70, dtype=synth.STATE)
st["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], axis=1)
st["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], axis=1)
eng.particles_set(st, prior)
a = synth.make_poses([[0, 0, 0]], [[0, 0, 0, 1]])
eng.particles_predict(a, a, 0.1, 10.0, 10.0)
sm = eng.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.05)
est = eng.particles_estimate(a, 0.2, 0.2)
eng.particles_resample(np.full(3, 0.01, np.float32), np.full(3, 0.01, np.float32), 0.3, seed=5)
out, p = eng.particles_get()
print("resident", sm["kept"], est["max_index"], round(float(p.sum()), 4))
raw = np.tile(np.concatenate([s["lik"], s["beam"]]), 20)
info = eng.scan_prepare(raw, engine.ScanParams(lik_num_points=50, beam_num_points=7, seed=3))
sm2 = eng.particles_measure_update_prepared(s["origins"], 0.0)
print("scan", info, sm2["kept"])
ns = eng.scan_sample_with_normal((0, 0, 0, 1), np.diag([0.6, 0.05, 0.02]), None, 50, 7, seed=3)
sm3 = eng.particles_measure_update_prepared(s["origins"], 0.0)
print("normal sampler", ns["n_lik"], ns["n_beam"], ns["rounds"], len(eng.scan_normals(0)[0]), sm3["kept"])
eng.close()
print("sanitize run complete")
