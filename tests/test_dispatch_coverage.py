"""The GPU dispatch matrix (test_gpu_dispatch_matrix.py) must reach every assembly kernel the host can select.  The
selection rules are restated in dispatch_scenes.expected_paths; this CPU test checks that the scene catalogue x switch
matrix covers all of them, and that every scene still lands on the cell it is named for."""
import pytest

import dispatch_scenes as D

# (K, dcmax, largest columns per image, structural cells it must have) per catalogue scene
SCENE_SHAPES = {
    "k3_dc7": (3, 9, 7, set()),
    "k4_dc8": (4, 10, 8, set()),
    "k5_dc7": (5, 11, 7, set()),
    "k8_dc8": (8, 14, 8, set()),
    "k12_dc8": (12, 18, 8, set()),
    "k8_dc14": (8, 14, 14, set()),
    "mixed_dc8": (8, 14, 8, {"mixed_models", "shared_and_per_image_cameras"}),
    "mixed_dc14": (8, 14, 14, {"mixed_models", "shared_and_per_image_cameras", "generic_walk_fast_and_generic_chunks"}),
    "pose_intr_only": (4, 10, 7,{"image_without_columns", "intrinsics_only_image", "pose_only_image", "partial_tvec_masks"}),
    "dup_obs": (4, 10, 8, {"same_image_non_self_pairs"}),
    "multi_chunk": (4, 10, 8, {"key_over_one_chunk", "image_over_one_chunk"}),
}


@pytest.fixture(scope="module")
def scenes():
    return {name: build() for name, build in D.SCENES.items()}


def _rows():
    for s in D.SCENES:
        for env in D.DENSE_ENVS:
            yield s, env, 0
    for s in D.SPARSE_SCENES:
        for env in D.SPARSE_ENVS:
            yield s, env, 3 if "PXR_PCG_SPARSE" in env else 0


def test_every_scene_lands_on_its_cell(scenes):
    assert set(SCENE_SHAPES) == set(D.SCENES)
    for name, (K, dcmax, dc_max, cells) in SCENE_SHAPES.items():
        sh = D.shape(scenes[name])
        assert (sh["K"], sh["dcmax"], sh["img_dc_max"]) == (K, dcmax, dc_max), name
        assert D.cells(scenes[name]) >= cells, name


def test_catalogue_and_switches_reach_every_assembly_kernel(scenes):
    reached = {}
    for s, env, ls in _rows():
        for k in D.expected_paths(scenes[s], env, linear_solver=ls):
            reached.setdefault(k, []).append((s, D.env_id(env)))
    assert set(reached) <= D.ALL_PATHS, set(reached) - D.ALL_PATHS
    assert set(reached) == D.ALL_PATHS, "never launched by the matrix: %s" % sorted(D.ALL_PATHS - set(reached))
    cells = set().union(*(D.cells(sc) for sc in scenes.values()))
    assert cells == D.ALL_CELLS, sorted(D.ALL_CELLS - cells)


def test_selection_rules_at_known_points(scenes):
    """spot checks of the restated rules against the shared-memory arithmetic of BA::build and BA::project"""
    p = D.expected_paths
    # K = 8 and 12: the staged build's 53 248 / 65 536 B exceed 48 KiB, so the unstaged chunked build runs
    assert "ba_build_kernel<true>/chunked" in p(scenes["k8_dc8"], {})
    assert "ba_build_kernel<true>/chunked" in p(scenes["k12_dc8"], {})
    assert "ba_build_staged_kernel" in p(scenes["k5_dc7"], {})
    assert "ba_build_kernel<true>/atomic" in p(scenes["k4_dc8"], {"PXR_BUILD_ATOMIC": "1"})
    # the projection's staged record fits for every model
    assert all("ba_project_staged_kernel" in p(sc, {}) for sc in scenes.values())
    # odd dcmax takes the 8-byte-gather staged walk
    assert "ba_schur_pairs_staged_kernel<false, 4>" in p(scenes["k3_dc7"], {"PXR_SCHUR_KERNEL": "staged"})
    assert "sp_schur_pairs_kernel<2>" in p(scenes["k5_dc7"], {"PXR_PCG_SPARSE": "1", "PXR_SCHUR_KERNEL": "staged"}, 3)
    # PXR_PCG_SPARSE means nothing for the exact solver; more than 8 columns never take a staged / tensor-core walk
    assert "ba_schur_pairs_mma_kernel<4, true>" in p(scenes["k4_dc8"], {"PXR_PCG_SPARSE": "1"}, 0)
    assert p(scenes["k8_dc14"], {"PXR_SCHUR_KERNEL": "mma"}) >= {"ba_schur_prep_kernel", "ba_schur_pairs_kernel<false>"}
