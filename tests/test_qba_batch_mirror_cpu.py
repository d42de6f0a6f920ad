"""The batched localization entry points (QueryBundleAdjuster.refine_multilevel_batch, QueryLocalizer.localize_batch)
without a device: the device entry points of `_engine` are replaced by the oracle as in test_mirror_with_oracle_solver,
`_engine.qba_run` by a loop of the oracle's BA solve over the per-query problems, and the batched calls must give what
a loop of the single-query calls gives."""
import numpy as np
import pytest

import oracle_lib as O
from pixsfm._pixsfm import _capi, _engine
from test_mirror_with_oracle_solver import oracle_engine  # noqa: F401  (fixture)


def _qba_run(batch, interp=None, options=None, ctx=None, capacity=0):
    interp = interp or _capi.default_interp()
    out, p0 = [], 0
    for k in range(batch.n_queries):
        b0, b1 = int(batch.obs_begin[k]), int(batch.obs_begin[k + 1])
        n = int(batch.patch_counts[k])
        r = dict(status=_capi.PXR_OK, num_residual_blocks=b1 - b0, initial_cost=0.0, final_cost=0.0, num_iterations=0,
                 num_successful_steps=0, num_unsuccessful_steps=0, termination_type=1, block_evaluations=0, iterations=[])
        if b1 > b0:
            m = b1 - b0
            prob = _capi.BAProblem(cam_model=[batch.cam_model[k]], cam_params=batch.cam_params[k:k + 1],
                                   cam_const_mask=[batch.cam_const_mask[k]], qvec=batch.qvec[k:k + 1], tvec=batch.tvec[k:k + 1],
                                   img_cam=[0], pose_const=[0], tvec_const_mask=[0], xyz=batch.xyz[b0:b1],
                                   point_const=np.ones(m, np.uint8), obs_img=np.zeros(m, np.int32),
                                   obs_pt=np.arange(m, dtype=np.int64), patches=np.ascontiguousarray(batch.patch_blocks[k]),
                                   corner=batch.corner[p0:p0 + n], scale=batch.scale[p0:p0 + n], refs=batch.refs[b0:b1],
                                   obs_patch=batch.obs_patch[b0:b1])
            s = O.ba_solve(prob, interp, options)
            batch.qvec[k], batch.tvec[k], batch.cam_params[k] = prob.qvec[0], prob.tvec[0], prob.cam_params[0]
            r.update({key: s[key] for key in ("initial_cost", "final_cost", "num_successful_steps",
                                               "num_unsuccessful_steps", "termination_type", "num_iterations")})
            r["iterations"] = s["iterations"]
        out.append(r)
        p0 += n
    return out, dict(n_waves=1, h2d_bytes=0.0, solve_time_s=0.0, total_time_s=0.0, kernel_launches=0, message="")


@pytest.fixture
def oracle_qba(oracle_engine, monkeypatch):  # noqa: F811
    monkeypatch.setattr(_engine, "qba_run", _qba_run)


def test_refine_multilevel_batch(oracle_qba):
    import test_gpu_qba_batch as T
    T.test_refine_multilevel_batch_matches_loop()


def test_localize_batch(oracle_qba):
    import test_gpu_qba_batch as T
    T.test_localize_batch_matches_localize()
