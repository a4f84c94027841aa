"""CPU: the training loop's pruning schedule (training.prune_milestones, prune_min_views, prune_max_outside): the
defaults, the refusals of check_config, and which checkpoint sizes resume accepts with pruning."""
import copy

import pytest

from dss_b200.training.config import DEFAULTS, GROW_K, check_cloud_size, check_config


def config(milestones, min_views=1, max_outside=0, grow=((), ()), n0=2000):
    cfg = copy.deepcopy(DEFAULTS)
    cfg["model"]["model_kwargs"]["n_points_per_cloud"] = n0
    tr = cfg["training"]
    tr["prune_milestones"], tr["prune_min_views"], tr["prune_max_outside"] = milestones, min_views, max_outside
    tr["grow_milestones"], tr["grow_points"] = list(grow[0]), list(grow[1])
    return cfg


def check(cfg):
    check_config(cfg, (512, 512), True)


def test_defaults_prune_nothing():
    tr = DEFAULTS["training"]
    assert tr["prune_milestones"] == [] and tr["prune_min_views"] == 1 and tr["prune_max_outside"] == 0
    check(copy.deepcopy(DEFAULTS))


@pytest.mark.parametrize("milestones, min_views, max_outside", [
    ([1], 1, 0), ([100, 200], 0, 3), ([5], 2, None), ([], 0, None), ((7, 9), 1, 0),
])
def test_accepted_schedules(milestones, min_views, max_outside):
    check(config(milestones, min_views, max_outside))


@pytest.mark.parametrize("milestones, min_views, max_outside, match", [
    ([200, 100], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    ([100, 100], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    ([0], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    ([-3], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    ([10.0], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    ([True], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    (["10"], 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    (10, 1, 0, "prune_milestones must be a list of strictly increasing integers >= 1"),
    ([10], -1, 0, "prune_min_views must be an integer >= 0"),
    ([10], 1.5, 0, "prune_min_views must be an integer >= 0"),
    ([10], None, 0, "prune_min_views must be an integer >= 0"),
    ([10], True, 0, "prune_min_views must be an integer >= 0"),
    ([10], 1, -1, "prune_max_outside must be an integer >= 0 or null"),
    ([10], 1, 0.5, "prune_max_outside must be an integer >= 0 or null"),
    ([10], 1, False, "prune_max_outside must be an integer >= 0 or null"),
    ([10], 0, None, "turn both of its tests off"),
])
def test_refused_schedules(milestones, min_views, max_outside, match):
    with pytest.raises(ValueError, match=match):
        check(config(milestones, min_views, max_outside))


def test_thresholds_are_checked_without_milestones():
    with pytest.raises(ValueError, match="prune_min_views"):
        check(config([], -2, 0))


def test_other_refusals_come_first():
    with pytest.raises(ValueError, match="image_size"):
        check_config(config([0]), (128, 128), True)
    with pytest.raises(ValueError, match="grow_milestones"):
        check(config([0], grow=([0], [4000])))


def ok(cfg, it, n):
    check_cloud_size(cfg, it, n)


def refused(cfg, it, n):
    with pytest.raises(ValueError, match="the checkpoint holds %d points after it=%d, but" % (n, it)):
        check_cloud_size(cfg, it, n)


def test_checkpoint_size_with_pruning_alone():
    cfg = config([100, 300])
    for it in (-1, 0, 99):                  # before the first prune: the initial size
        ok(cfg, it, 2000)
        refused(cfg, it, 1999)
    for it in (100, 250, 300, 10 ** 6):     # after a prune: anything from GROW_K + 1 to the size
        for n in (GROW_K + 1, 1000, 2000):
            ok(cfg, it, n)
        for n in (GROW_K, 1, 2001):
            refused(cfg, it, n)


def test_checkpoint_size_with_pruning_and_growth():
    cfg = config([100, 200, 400], grow=([200, 300], [4000, 8000]))
    for it, n in ((99, 2000), (100, 17), (150, 1999), (150, 2000), (200, 4000), (299, 4000), (300, 8000),
                  (399, 8000), (400, 8000), (400, 123), (10 ** 6, 7999)):
        ok(cfg, it, n)
    for it, n in ((99, 1500), (150, 2001), (150, 16),
                  (200, 3999), (200, 2000),     # a prune and a growth on one iteration: the growth comes last
                  (250, 2000), (300, 4000), (399, 7999), (400, 8001)):
        refused(cfg, it, n)
    with pytest.raises(ValueError, match="gives 17 to 2000 there"):
        check_cloud_size(cfg, 150, 2001)
    with pytest.raises(ValueError, match="gives 4000 there"):
        check_cloud_size(cfg, 200, 2000)


def test_a_small_cloud_that_was_never_pruned_resumes():
    # a prune leaves a cloud of GROW_K or fewer points as it is: its size stays acceptable after the milestone
    cfg = config([10], n0=GROW_K)
    ok(cfg, 20, GROW_K)
    refused(cfg, 20, GROW_K - 1)


def test_checkpoint_size_without_pruning_is_unchanged():
    # without a pruning schedule the growth rules alone apply, and without either any size resumes
    refused(config([], grow=([300], [4000])), 350, 3000)
    ok(config([], grow=([300], [4000])), 350, 4000)
    for n in (10, 2000, 123456):
        ok(config([]), 500, n)
