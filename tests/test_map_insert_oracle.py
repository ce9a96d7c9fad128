"""The CPU oracle's map_insert (lk_map_insert restated: calcBodyCov, the placement of KILO.cc:216-228 at explicit poses,
UpdateVoxelMap set by set) against the reference: the fixtures tests/golden/ref_map_insert.npz made by the reference
itself (tests/golden/make_ref_map_insert_golden.py), and random poses and covariances against the compiled reference
where it is available."""
import os

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import general_prior as gp
import lko_insert
import lkref_insert
import map_insert_cases as mic
import mapcmp
from legkilo_b200 import abi, synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_map_insert.npz")


def fixture(name):
    """Case `name` of the fixture: (cfg, call buffers, digest of the start map or None, digest after the insert)."""
    z = np.load(GOLD)
    c = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}
    return abi.CONFIGS["leg_fusion"], c, c.pop("map0", None), c.pop("map1")


@pytest.mark.parametrize("name", mic.NAMES)
def test_oracle_matches_reference_fixture(name):
    cfg, c, map0, map1 = fixture(name)
    blob0 = mic.start_blob(cfg, c)
    assert (blob0 is None) == (map0 is None)
    if blob0 is not None:
        mapcmp.compare_digest(map0, blob0)
    st_ = mapcmp.compare_digest(map1, mic.oracle_insert(cfg, blob0, *mic.call(c)))
    assert st_["planes"] > 100, st_


def test_fixture_cases_are_the_generator_cases():
    """The committed buffers are the ones tests/map_insert_cases.py makes (the device tests rebuild them from there)."""
    for name in mic.NAMES:
        _, c, _, _ = fixture(name)
        _, c2 = mic.case(name)
        assert set(c) == set(c2), name
        for k in c:
            np.testing.assert_array_equal(np.asarray(c2[k]).reshape(c[k].shape), c[k], err_msg=f"{name} {k}")


def _random_call(seed, n_sets, cfg_name):
    """A few box-room scans split into n_sets sets at arbitrary boundaries (some empty), each at a pose drawn anywhere
    (uniform attitude, positions within +-3 km) with random SPD covariance blocks, on top of the room's first-frame map."""
    cfg = abi.CONFIGS[cfg_name]
    g = synth.rng(seed)
    G = gp.so3_uniform(g)
    pG = g.uniform(-3000.0, 3000.0, 3)
    sc, pw, pb = gp.map_cloud(cfg, G, pG)
    pts = np.concatenate([gp.room_scan(cfg, sc, seed + 1 + i, False, n_az=60) for i in range(2)])
    cuts = np.sort(g.integers(0, len(pts) + 1, n_sets - 1))
    so = np.concatenate([[0], cuts, [len(pts)]]).astype(np.uint32)
    rot = np.array([G @ synth.exp_so3(0.003 * g.standard_normal(3)) for _ in range(n_sets)])
    pos = pG + 0.03 * g.standard_normal((n_sets, 3))
    covs = []
    for scale in (3e-3, 0.03):
        A = g.standard_normal((n_sets, 3, 3))
        covs.append(scale ** 2 * (A @ A.transpose(0, 2, 1) / 3.0 + 0.1 * np.eye(3)))
    return cfg, (pw, pb, G), (pts, so, rot, pos, covs[0], covs[1])


@pytest.mark.skipif(not lkref_insert.available(), reason="needs oracle/_ref/liblkref_insert.so or /root/reference")
@settings(max_examples=6, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
@given(seed=st.integers(9600, 9999), n_sets=st.integers(1, 7), cfg_name=st.sampled_from(["leg_fusion", "hilti", "diter"]),
       on_map=st.booleans())
def test_oracle_matches_reference_random(seed, n_sets, cfg_name, on_map):
    cfg, (pw, pb, G), args = _random_call(seed, n_sets, cfg_name)
    o, r = lko_insert.Oracle(cfg), lkref_insert.Reference(cfg)
    if on_map:
        rc, pc = gp.map_covs(G)
        o.build_voxel_map(pw, pb, R=G, rot_cov=rc, pos_cov=pc)
        r.build_voxel_map(pw, pb, R=G, rot_cov=rc, pos_cov=pc)
    o.map_insert(*args)
    r.map_insert(*args)
    st_ = mapcmp.compare_blobs(r.map_export(), o.map_export())
    assert st_["points"] > 0, st_
