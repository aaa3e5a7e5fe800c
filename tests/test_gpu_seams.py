"""The sharded step on one GPU against the restatement (oracle/cityflow_oracle.cpp), on irregular networks, at the seam's
edges and under cuts other than column strips.

A loop-back group (cityflow_b200.capi.CShardGroup) runs the ranks of one simulation on one GPU with the real seam kernels
of csrc/device_shard.cuh: 128-thread blocks, one warp per seam lane in k_xchg_movers, grid-stride loops, the block ticket
of shardLastBlock.  The emulated device of tests/test_cpu.py runs every block as one warp, so the block and grid shapes
are only ever run here.  Every step, every running vehicle -- every field and every drivable's list order -- and the
ranks' summed counters must equal the restatement's (edgenet.group_vs_restatement).
"""
import os
import time

import pytest

pytestmark = pytest.mark.gpu

# device_sim.cu: k_xchg_movers runs at most 64 blocks of 4 warps (one warp per seam lane), k_xchg_tails 16 blocks of 128
# threads (one thread per seam lane); a rank with more seam lanes than that goes round the grid-stride loops.
MOVER_WARPS = 64 * 4
TAIL_THREADS = 16 * 128


def _run(cfg, world, steps, owners=None):
    import edgenet
    from cityflow_b200.capi import CShardGroup
    reach = edgenet.SeamReach(edgenet.loader_tables(cfg), edgenet.partition(cfg, world, owners))
    grp = CShardGroup(cfg, world, owners)
    t0 = time.time()
    ora = edgenet.group_vs_restatement(grp, cfg, steps, reach)
    grp.close()
    print("%s, %d ranks, %s: %d steps in %.1f s, %d vehicles at the end; %s" %
          (os.path.basename(cfg), world, "column strips" if owners is None else "cut by owners", steps, time.time() - t0,
           ora.vehicle_count(), reach))
    return ora, reach


def test_checkerboard_cut_past_the_seam_kernels_grid_caps(tmp_path):
    """A dense 20x20 grid cut as a checkerboard over two ranks: every road is a seam road, so each rank feeds and owns
    over 2500 seam lanes -- more than k_xchg_movers' 256 warps and k_xchg_tails' 2048 threads, whose loops go round."""
    import edgenet
    from cityflow_b200 import scenario
    cfg = scenario.make_grid_scenario(str(tmp_path), 20, 20, dense=dict(frac=1.0, interval=6.0, seed=7), name="cb20")
    owners = edgenet.checkerboard_owners(cfg)
    reach = edgenet.SeamReach(edgenet.loader_tables(cfg), edgenet.partition(cfg, 2, owners))
    print("20x20 checkerboard: seam lanes fed per rank %s, owned per rank %s" % (reach.feeds, reach.owns))
    assert min(reach.feeds + reach.owns) > TAIL_THREADS > MOVER_WARPS
    ora, reach = _run(cfg, 2, 200, owners)
    assert ora.vehicle_count() > 5000 and sum(t for t, _ in reach.crossed.values()) > 1000, str(reach)


def test_checkerboard_cut_of_a_small_grid(tmp_path):
    """The dense 4x4 checkerboard of the emulated suite, on the GPU."""
    import edgenet
    from cityflow_b200 import scenario
    cfg = scenario.make_grid_scenario(str(tmp_path), 4, 4, dense=dict(frac=1.0, interval=3.0, seed=4), name="cb")
    _, reach = _run(cfg, 2, 250, edgenet.checkerboard_owners(cfg))
    assert reach.spawns > 0 and reach.finishes > 0 and reach.foreign_blockers > 0, str(reach)


def _randnet_cfg(seed, interval, directory):
    import randnet
    from cityflow_b200 import scenario
    net = randnet.random_roadnet(seed)
    return scenario.write_scenario(directory, net, randnet.random_flows(net, seed + 100), seed=seed, interval=interval,
                                   name="rand%d" % seed)


@pytest.mark.parametrize("seed,interval", [(3, 0.5), (6, 0.25)])
def test_fuzzed_networks_column_strips_and_scattered_cuts(seed, interval, tmp_path):
    """Two tests/randnet.py networks, each cut into three column strips and scattered over four ranks."""
    import edgenet
    cfg = _randnet_cfg(seed, interval, str(tmp_path))
    _, strips = _run(cfg, 3, 250)
    _, scattered = _run(cfg, 4, 250, edgenet.scattered_owners(cfg, 4, seed * 10 + 4))
    assert max(scattered.neighbours) >= 3 and scattered.foreign_blockers > 0, str(scattered)
    assert strips.spawns > 0 and scattered.spawns > 0


def test_long_queue_cut_between_a_and_b(tmp_path):
    """long_queue in two column strips: the seam lane A -> B queues end to end against B's red, and A's laneLinks wait
    on its ghost tail."""
    import edgenet
    cfg = edgenet.write("long_queue", str(tmp_path))
    _, reach = _run(cfg, 2, 700)
    assert reach.max_queue > 0.97 and reach.halted_feeding > 0, str(reach)


@pytest.mark.parametrize("world", [2, 4])
def test_star_cut_at_the_joining_road(world, tmp_path):
    """star in column strips: at two ranks the joining road is the seam in both directions; at four, two ranks own no
    real intersection."""
    import edgenet
    cfg = edgenet.write("star", str(tmp_path))
    _, reach = _run(cfg, world, 400)
    if world == 2:
        assert reach.max_movers >= 2, str(reach)
    else:
        assert len(reach.empty_ranks) == 2, str(reach)


def test_mover_message_at_entrant_capacity(tmp_path):
    """merge_16 in two column strips: sixteen tied vehicles enter the seam lane I -> J in one step, one full mover
    message (ENT_CAP records) for the owner's k_move to rank by priority."""
    import edgenet
    cfg = edgenet.write("merge_16", str(tmp_path))
    ora, reach = _run(cfg, 2, 200)
    assert reach.max_movers == 16 and ora.tie_reach()["groups"].get(16, 0) >= 1, (str(reach), ora.tie_reach())


def test_scattered_cut_over_the_staged_exchange(tmp_path, monkeypatch):
    """A scattered cut exchanging through the staged path (k_pack_* / k_unpack_* / k_seal_blk / k_apply_blk, moved
    between the ranks by device copies): CITYFLOW_B200_SHARD_TRANSPORT=nccl at the group's creation."""
    import edgenet
    from cityflow_b200.capi import CShardGroup
    cfg = _randnet_cfg(5, 1.0, str(tmp_path))
    owners = edgenet.scattered_owners(cfg, 3, 53)
    reach = edgenet.SeamReach(edgenet.loader_tables(cfg), edgenet.partition(cfg, 3, owners))
    monkeypatch.setenv("CITYFLOW_B200_SHARD_TRANSPORT", "nccl")
    grp = CShardGroup(cfg, 3, owners)
    monkeypatch.delenv("CITYFLOW_B200_SHARD_TRANSPORT")
    ora = edgenet.group_vs_restatement(grp, cfg, 250, reach)
    grp.close()
    print("staged exchange, scattered cut over 3 ranks: %d vehicles at the end; %s" % (ora.vehicle_count(), reach))
    assert reach.foreign_blockers > 0 and sum(t for t, _ in reach.crossed.values()) > 0, str(reach)
