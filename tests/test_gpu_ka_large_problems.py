"""Keypoint-adjustment problems of more than 80 variable keypoints on the GPU, against the oracle (which solves every
problem densely): many small components in one problem, a problem whose workspace does not fit in shared memory and
runs off chip, the per-component limit, the `low_memory` preset's topological-reference KA, `split_in_subproblems:
False` and `run_subset`."""
import re

import numpy as np
import pytest

import oracle_lib as O
from pixsfm import base, configs, features, keypoint_adjustment as ka_pkg
from pixsfm._pixsfm import _capi, _engine
from pixsfm._pixsfm import _keypoint_adjustment as ka
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu


def _id(v):
    return v.__name__ if isinstance(v, type) else str(v)


def _merge(scenes):
    """the node and edge arrays of several synthetic KA scenes as one scene (no edge between them)"""
    out = {k: [] for k in ("keypoints", "node_image", "node_feature", "edge_src", "edge_dst", "edge_sim", "patches",
                           "corner", "scale")}
    n = 0
    for sc in scenes:
        for k in out:
            out[k].append(sc[k] + n if k in ("edge_src", "edge_dst") else sc[k])
        n += len(sc["keypoints"])
    return {k: np.concatenate(v) for k, v in out.items()}


def _problem(parts, bound=4.0):
    """one KAProblem from (scene, max keypoints per problem) parts, each packed on its own (first-fit decreasing, as
    keypoint_adjustment/main.py does) into problems of its own; featuremetric intra-track edges, roots constant"""
    kps, const, patches, corner, scale, es, ed, ew, ep = [], [], [], [], [], [], [], [], []
    n = n_prob = 0
    for sc, max_per_problem in parts:
        tl, _, roots = _engine.graph_labels(sc["node_image"], sc["edge_src"], sc["edge_dst"], sc["edge_sim"])
        plabels, n_p = _engine.ka_problem_labels(tl, max_per_problem)
        intra = tl[sc["edge_src"]] == tl[sc["edge_dst"]]
        s, d = sc["edge_src"][intra], sc["edge_dst"][intra]
        es.append(s + n); ed.append(d + n); ew.append(sc["edge_sim"][intra]); ep.append(plabels[s] + n_prob)
        kps.append(sc["keypoints"]); const.append(roots); patches.append(sc["patches"])
        corner.append(sc["corner"]); scale.append(sc["scale"])
        n += len(sc["keypoints"]); n_prob += n_p
    es, ed, ew, ep = (np.concatenate(v) for v in (es, ed, ew, ep))
    order = np.argsort(ep, kind="stable")
    roots = np.concatenate(const)
    prob = _capi.KAProblem(keypoints=np.concatenate(kps), kp_const=roots, edge_src=es[order], edge_dst=ed[order],
                           edge_weight=ew[order], edge_problem=ep[order], n_problems=n_prob,
                           patches=np.ascontiguousarray(np.concatenate(patches)), corner=np.concatenate(corner),
                           scale=np.concatenate(scale), bound=bound, patches_are_sparse=True)
    return prob, roots.astype(bool)


def _variable_per_problem(prob):
    var = np.zeros(prob.n_problems, np.int64)
    for p in range(prob.n_problems):
        m = prob.edge_problem == p
        ends = np.unique(np.concatenate([prob.edge_src[m], prob.edge_dst[m]]))
        var[p] = int(np.sum(prob.kp_const[ends] == 0))
    return var


def _offchip(summary):
    m = re.search(r"(\d+) with an off-chip workspace", summary["message"])
    assert m, summary["message"]
    return int(m.group(1))


def _compare(prob, ic, so, roots):
    """GPU vs oracle at the tolerances of test_gpu_ka.py; -> the GPU summary"""
    p_cpu, p_gpu = prob.copy(), prob.copy()
    c0, c1 = O.ka_solve(p_cpu, ic, so)
    s = _engine.ka_run(p_gpu, ic, so)
    assert abs(s["initial_cost"] - c0) <= 1e-9 * c0
    assert abs(s["final_cost"] - c1) <= 1e-6 * c1
    assert c1 < c0
    assert np.abs(p_gpu.keypoints - p_cpu.keypoints).max() < 1e-5
    assert np.array_equal(p_gpu.keypoints[roots], prob.keypoints[roots])
    assert np.abs(p_gpu.keypoints[~roots] - prob.keypoints[~roots]).max() > 1e-3
    return s


def _mixed_tracks(dtype, seed, n_tracks=50):
    """tracks of 3, 4, 5 and 6 keypoints"""
    return _merge([synthetic.make_ka_scene(n_images=8, n_tracks=n_tracks, track_len=L, channels=128, seed=seed + L,
                                           kp_sigma=0.7, dtype=dtype) for L in (3, 4, 5, 6)])


# ---- 1. many small components in problems of a few hundred variable keypoints

@pytest.mark.parametrize("variant", ["bounded_cauchy", "unbounded_cauchy", "bounded_trivial"])
@pytest.mark.parametrize("dtype,fs", [(np.float64, 0), (np.float16, 1), (np.float16, 0)], ids=_id)
def test_many_small_components(dtype, fs, variant):
    prob, roots = _problem([(_mixed_tracks(dtype, seed=31), 310)])
    var = _variable_per_problem(prob)
    assert prob.n_problems >= 3 and var.min() >= 150 and var.max() <= 400, var
    so = _capi.default_ka_options()
    if variant == "unbounded_cauchy":
        prob.bound = -1.0
        prob.patches_are_sparse = False        # dense maps and bound <= 0: no box constraint at all
    elif variant == "bounded_trivial":
        so = _capi.default_ka_options(loss_type=0, loss_scale=1.0)
    s = _compare(prob, _capi.default_interp(use_float_simd=fs), so, roots)
    assert _offchip(s) == 0                    # components of 2-5 variable keypoints: a few tens of KB, on chip


# ---- 2. a problem whose workspace does not fit in shared memory, launched with small on-chip problems

@pytest.mark.parametrize("dtype,fs", [(np.float64, 0), (np.float16, 1)], ids=_id)
def test_offchip_problem_among_onchip_problems(dtype, fs):
    # three tracks seen in 81 images: 240 variable keypoints in three 160-scalar components, 3 x 12 880 doubles per
    # matrix and 656 640 B of workspace in all
    big = synthetic.make_ka_scene(n_images=81, n_tracks=3, track_len=81, channels=128, seed=5, kp_sigma=0.7,
                                  dtype=dtype, extra_edge_prob=0.05)
    small = synthetic.make_ka_scene(n_images=6, n_tracks=30, track_len=4, channels=128, seed=6, kp_sigma=0.7,
                                    dtype=dtype)
    prob, roots = _problem([(big, 1000), (small, 20)])
    var = _variable_per_problem(prob)
    assert var[0] == 240 and prob.n_problems >= 6 and var[1:].max() <= 20
    s = _compare(prob, _capi.default_interp(use_float_simd=fs), _capi.default_ka_options(), roots)
    assert _offchip(s) == 1


# ---- 3. the per-component limit inside a large problem

def test_component_of_81_variable_keypoints_is_refused():
    sc = _merge([synthetic.make_ka_scene(n_images=82, n_tracks=1, track_len=82, channels=128, seed=7, kp_sigma=0.7,
                                         dtype=np.float64, extra_edge_prob=0.05),
                 synthetic.make_ka_scene(n_images=6, n_tracks=40, track_len=4, channels=128, seed=8, kp_sigma=0.7,
                                         dtype=np.float64)])
    prob, _ = _problem([(sc, 1000)])
    assert prob.n_problems == 1 and _variable_per_problem(prob)[0] == 81 + 120
    before = prob.keypoints.copy()
    with pytest.raises((ValueError, _capi.PxrError), match="80 supported"):
        _engine.ka_run(prob, _capi.default_interp(), _capi.default_ka_options())
    assert np.array_equal(prob.keypoints, before)


# ---- 4. and 5. through the Python surface

def _graph_scene(n_images, n_tracks, ps, seed, track_len=4):
    sc = synthetic.make_ka_scene(n_images=n_images, n_tracks=n_tracks, track_len=track_len, channels=128, ps=ps,
                                 seed=seed, kp_sigma=1.0)
    g = base.Graph()
    names = ["im%d" % i for i in range(n_images)]
    keypoints = {names[i]: np.ascontiguousarray(sc["keypoints"][sc["node_image"] == i]) for i in range(n_images)}
    for n in range(len(sc["node_image"])):
        g.add_node(names[sc["node_image"][n]], int(sc["node_feature"][n]))
    for e in range(len(sc["edge_src"])):
        g.add_edge(g.nodes[sc["edge_src"][e]], g.nodes[sc["edge_dst"][e]], sc["edge_sim"][e])
    fm = features.FeatureManager([128], np.float16)
    for i in range(n_images):
        m = np.where(sc["node_image"] == i)[0]
        fm.fset(0).emplace(names[i], features.FeatureMap(np.ascontiguousarray(sc["patches"][m]),
                                                          sc["node_feature"][m].tolist(), sc["corner"][m],
                                                          {"scale": sc["scale"][m[0]], "is_sparse": True}))
    track_labels = base.compute_track_labels(g)
    root_labels = base.compute_root_labels(g, track_labels, base.compute_score_labels(g, track_labels))
    return g, keypoints, fm, track_labels, root_labels


@pytest.fixture
def ka_calls(monkeypatch):
    """every pxr_ka_run call the Python layer makes: (problem before, interp, options, problem after, summary)"""
    calls, run = [], _engine.ka_run

    def spy(problem, interp=None, options=None, ctx=None):
        before = problem.copy()
        s = run(problem, interp, options, ctx)
        calls.append((before, interp, options, problem.copy(), s))
        return s
    monkeypatch.setattr(_engine, "ka_run", spy)
    return calls


def _against_oracle(call):
    before, ic, so, after, s = call
    p_cpu = before.copy()
    c0, c1 = O.ka_solve(p_cpu, ic, so)
    assert abs(s["initial_cost"] - c0) <= 1e-9 * c0
    assert abs(s["final_cost"] - c1) <= 1e-6 * c1 and c1 < c0
    assert np.abs(after.keypoints - p_cpu.keypoints).max() < 1e-5


def _check_roots(g, keypoints, before, root_labels):
    for n, node in enumerate(g.nodes):
        name = g.image_id_to_name[node.image_id]
        d = np.abs(keypoints[name][node.feature_idx] - before[name][node.feature_idx]).max()
        assert (d == 0.0) if root_labels[n] else (d > 0.0)


def _low_memory_ka():
    conf = configs.parse_config_path("low_memory")["mapping"]["KA"]
    assert conf["strategy"] == "topological_reference" and conf["max_kps_per_problem"] == 1000
    assert conf["optimizer"]["bound"] == 2.0
    return conf


def test_low_memory_preset_matches_oracle(ka_calls):
    g, keypoints, fm, tl, rl = _graph_scene(n_images=6, n_tracks=100, ps=8, seed=41)
    before = {k: v.copy() for k, v in keypoints.items()}
    out = ka_pkg.KeypointAdjuster.create(_low_memory_ka()).refine_multilevel(keypoints, fm, g, tl, rl)
    assert len(ka_calls) == 1
    prob = ka_calls[0][0]
    assert prob.n_problems == 1 and prob.bound == 2.0 and prob.patches[0].shape[:2] == (8, 8)
    assert _variable_per_problem(prob)[0] == 300
    _against_oracle(ka_calls[0])
    assert out["summary"][0].num_residual_blocks == len(g.nodes) - int(np.sum(rl))
    _check_roots(g, keypoints, before, rl)


def test_low_memory_preset_in_bins_of_1000(ka_calls):
    g, keypoints, fm, tl, rl = _graph_scene(n_images=12, n_tracks=600, ps=8, seed=43)
    before = {k: v.copy() for k, v in keypoints.items()}
    out = ka_pkg.KeypointAdjuster.create(_low_memory_ka()).refine_multilevel(keypoints, fm, g, tl, rl)
    s = out["summary"][0]
    prob, summary = ka_calls[0][0], ka_calls[0][4]
    var = _variable_per_problem(prob)
    assert prob.n_problems == 3 and var.max() >= 700, var
    assert _offchip(summary) == 0              # ~750 singleton components: 156 KB of shared memory
    assert s.final_cost < s.initial_cost
    assert s.num_residual_blocks == len(g.nodes) - int(np.sum(rl))
    _check_roots(g, keypoints, before, rl)


@pytest.mark.parametrize("how", ["adjuster", "run_without_labels", "run_subset"])
def test_one_problem_over_the_whole_graph_matches_oracle(ka_calls, how):
    g, keypoints, fm, tl, rl = _graph_scene(n_images=6, n_tracks=60, ps=16, seed=45)
    before = {k: v.copy() for k, v in keypoints.items()}
    if how == "adjuster":
        ka_pkg.KeypointAdjuster.create({"split_in_subproblems": False}).refine_multilevel(keypoints, fm, g, tl, rl)
    else:
        setup = ka.KeypointAdjustmentSetup()
        setup.set_masked_nodes_constant(g, rl)
        opt = ka.FeatureMetricKeypointOptimizer({"bound": 4.0}, setup, {})
        if how == "run_without_labels":
            opt.run(keypoints, g, tl, rl, fm.fset(0))
        else:
            opt.run_subset(range(len(g.nodes)), keypoints, g, tl, rl, fm.fset(0))
    assert len(ka_calls) == 1
    prob = ka_calls[0][0]
    assert prob.n_problems == 1 and _variable_per_problem(prob)[0] == 180
    _against_oracle(ka_calls[0])
    assert _offchip(ka_calls[0][4]) == 0
    _check_roots(g, keypoints, before, rl)


def test_one_problem_past_shared_memory(ka_calls):
    """1 200 singleton components (topological reference) in one problem: 1 200 x 26 + 20 doubles, more than the
    227 KB of shared memory one H100 block can have, so the workspace is in global memory"""
    g, keypoints, fm, tl, rl = _graph_scene(n_images=12, n_tracks=400, ps=8, seed=47)
    before = {k: v.copy() for k, v in keypoints.items()}
    conf = dict(_low_memory_ka(), split_in_subproblems=False)
    out = ka_pkg.KeypointAdjuster.create(conf).refine_multilevel(keypoints, fm, g, tl, rl)
    s = out["summary"][0]
    prob, summary = ka_calls[0][0], ka_calls[0][4]
    assert prob.n_problems == 1 and _variable_per_problem(prob)[0] == 1200
    assert _offchip(summary) == 1
    assert s.final_cost < s.initial_cost
    _check_roots(g, keypoints, before, rl)
