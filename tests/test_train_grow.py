"""CPU: the training loop's growth schedule (training.grow_milestones / grow_points): the refusals of check_config, the
cloud's size at an iteration, and the refusal of a checkpoint whose size the schedule does not give."""
import copy

import pytest

from dss_b200.training.config import DEFAULTS, GROW_K, check_cloud_size, check_config, cloud_size


def config(milestones, points, n0=2000):
    cfg = copy.deepcopy(DEFAULTS)
    cfg["model"]["model_kwargs"]["n_points_per_cloud"] = n0
    cfg["training"]["grow_milestones"], cfg["training"]["grow_points"] = milestones, points
    return cfg


def check(cfg):
    check_config(cfg, (512, 512), True)


def test_defaults_grow_nothing():
    assert DEFAULTS["training"]["grow_milestones"] == [] and DEFAULTS["training"]["grow_points"] == []
    cfg = copy.deepcopy(DEFAULTS)
    check(cfg)
    assert [cloud_size(cfg, it) for it in (-1, 0, 10 ** 6)] == [8000] * 3


def test_accepted_schedules():
    check(config([300, 600], [4000, 8000]))
    check(config([1], [2001]))
    check(config([5], [100], n0=GROW_K + 1))          # the smallest cloud upsample_points grows with k = 16


@pytest.mark.parametrize("milestones, points, match", [
    ([300], [4000, 8000], "1 entries and training.grow_points 2"),
    ([300, 600], [4000], "2 entries and training.grow_points 1"),
    ([600, 300], [4000, 8000], "grow_milestones must be strictly increasing integers >= 1"),
    ([300, 300], [4000, 8000], "grow_milestones must be strictly increasing integers >= 1"),
    ([0, 300], [4000, 8000], "grow_milestones must be strictly increasing integers >= 1"),
    ([-5], [4000], "grow_milestones must be strictly increasing integers >= 1"),
    ([300.0], [4000], "grow_milestones must be strictly increasing integers >= 1"),
    ([True], [4000], "grow_milestones must be strictly increasing integers >= 1"),
    (["300"], [4000], "grow_milestones must be strictly increasing integers >= 1"),
    ([300, 600], [8000, 4000], "grow_points must be strictly increasing integers"),
    ([300, 600], [4000, 4000], "grow_points must be strictly increasing integers"),
    ([300], [4000.5], "grow_points must be strictly increasing integers"),
    ([300], [2000], r"grow_points must start above model.model_kwargs.n_points_per_cloud \(2000\)"),
    ([300], [1000], r"grow_points must start above model.model_kwargs.n_points_per_cloud \(2000\)"),
    (300, 4000, "must be lists"),
])
def test_refused_schedules(milestones, points, match):
    with pytest.raises(ValueError, match=match):
        check(config(milestones, points))


@pytest.mark.parametrize("n0", [GROW_K, 10, 9])
def test_refused_initial_cloud_that_cannot_grow(n0):
    with pytest.raises(ValueError, match="n_points_per_cloud = %d points cannot grow" % n0):
        check(config([10], [1000], n0=n0))


def test_other_refusals_come_first():
    # the existing refusals keep their order: a growth schedule is checked last
    cfg = config([300], [1000])
    with pytest.raises(ValueError, match="image_size"):
        check_config(cfg, (128, 128), True)


def test_cloud_size_at_an_iteration():
    cfg = config([300, 600], [4000, 8000])
    sizes = {it: cloud_size(cfg, it) for it in (-1, 0, 1, 299, 300, 301, 599, 600, 601, 10 ** 6)}
    assert sizes == {-1: 2000, 0: 2000, 1: 2000, 299: 2000, 300: 4000, 301: 4000, 599: 4000, 600: 8000, 601: 8000,
                     10 ** 6: 8000}


def test_checkpoint_size_against_the_schedule():
    cfg = config([300, 600], [4000, 8000])
    for it, n in ((-1, 2000), (129, 2000), (299, 2000), (300, 4000), (599, 4000), (600, 8000), (900, 8000)):
        check_cloud_size(cfg, it, n)
    for it, n in ((299, 4000), (300, 2000), (600, 4000), (129, 8000)):
        with pytest.raises(ValueError, match="the checkpoint holds %d points after it=%d, but .* gives %d there"
                                             % (n, it, cloud_size(cfg, it))):
            check_cloud_size(cfg, it, n)
    # an edited n_points_per_cloud is refused before the first milestone too
    with pytest.raises(ValueError, match="holds 2000 points after it=10"):
        check_cloud_size(config([300], [4000], n0=3000), 10, 2000)


def test_checkpoint_size_without_a_schedule_is_free():
    # as before growth existed: a checkpoint's cloud is taken at whatever size it has
    cfg = config([], [])
    for n in (10, 2000, 123456):
        check_cloud_size(cfg, 500, n)
