"""Handles that share a K1 kernel. K1 is one kernel per (kind, visibility form, buffers per warp or window layout), and
every id of a kind (every RoomGrid and BabyAI id) reaches the same one at its own geometry. Its dynamic shared-memory
limit (cudaFuncAttributeMaxDynamicSharedMemorySize) belongs to that kernel, not to a handle: a training process that
holds a training env and an eval env of another size, or a curriculum of sizes, steps a handle after a later mg_create
of the same kernel. Every step here is compared bit for bit with the oracle: image, direction, reward bits,
terminated and truncated, then grid, agent, rng and pending.

The cases are chosen with a mirror of configure_step's arithmetic (step_smem_bytes and its warp search): had mg_create
set the limit to what ITS geometry needs at its largest warp count, the handle created last would leave a limit below
the plan.smem of the handle created first, and launching that plan would be refused."""
import gc
import re
import threading
import time

import numpy as np
import pytest
import torch

import hash_support as hs
from babyai_oracle import BabyAIOracle
from babyai_pickup_oracle import PickupOracle
from minigrid_b200 import MinigridVecEnv, specs
from oracle.oracle import OracleVecEnv
from test_gpu_launch_chains import check_outputs, check_state, engine_outputs, first_diff, inject_ends, random_actions

pytestmark = pytest.mark.gpu

PLAN_RE = re.compile(r"K1 plan: layout=(\d+), (\d+) warps/CTA, vis=(\d+), nbuf=(\d+), (\d+) CTA/SM, grid=(\d+), smem=(\d+) B, "
                     r"tiles=(\d+)")
TILED, WINDOW = 0, 1
VIS_NONE, VIS_ALU, VIS_TBL = 0, 1, 2


@pytest.fixture(autouse=True)
def _knobs(monkeypatch):
    for knob in ("MINIGRID_B200_CFG", "MINIGRID_B200_GRID", "MINIGRID_B200_LAYOUT", "MINIGRID_B200_HOTFIRST"):
        monkeypatch.delenv(knob, raising=False)
    monkeypatch.setenv("MINIGRID_B200_VERBOSE", "1")


# ---- a mirror of configure_step's shared-memory arithmetic (mg_common.cuh: make_geom; mg_step_kernel.cuh; mg_step.cu) ----
K1_SMEM_MAX = 227 * 1024 - 1024  # the bound of configure_step's warp search
OBS_TILE_BYTES, VIS_TBL_BYTES, ORDER_CAP = 147 * 32, 128 * 128 * 2, 1024
ALL_IDS = {**specs.REGISTRY, **specs.BABYAI_REGISTRY, **specs.BABYAI_PICKUP_PUTNEXT_REGISTRY}


def words_per_env(W, H, layout):
    lsw_r, lsw_c, ring = (W + 3) >> 2, (H + 3) >> 2, 1 if layout == TILED else 3
    off_c = (H + 2 * ring) * lsw_r
    if layout == TILED:
        return off_c + (W + 2 * ring) * lsw_c
    return (((off_c + 3) & ~3) + (W + 2 * ring) * lsw_c + 3) & ~3


def layout_of(spec):
    """mg_create's rule: tiles of more than 512 bytes per env go to the window layout; Dynamic-Obstacles always tiled."""
    if spec.kind == specs.KIND_DYNOBS:
        return TILED
    return WINDOW if words_per_env(spec.width, spec.height, TILED) * 4 > 512 else TILED


def step_buf_bytes(W, H, layout):
    b = max(words_per_env(W, H, layout) * 128 if layout == TILED else 0, OBS_TILE_BYTES)
    return (b + 127) & ~127


def step_smem_bytes(W, H, layout, vis, warps, nbuf):
    return 1024 + (VIS_TBL_BYTES if vis == VIS_TBL else 0) + warps * nbuf * step_buf_bytes(W, H, layout) + 16 * warps + 32 + 2 * ORDER_CAP


def search_warps(W, H, layout, vis, nbuf):
    """configure_step's largest warp count: the variant's __launch_bounds__ cap, or fewer while the block exceeds the bound."""
    cap = 20 if (nbuf == 2 or layout == WINDOW) else 28
    return next(w for w in range(cap, 0, -1) if step_smem_bytes(W, H, layout, vis, w, nbuf) <= K1_SMEM_MAX)


def old_limit(spec, layout, vis, nbuf):
    """The limit mg_create used to leave on the kernel: what this geometry needs at its largest warp count."""
    return step_smem_bytes(spec.width, spec.height, layout, vis, search_warps(spec.width, spec.height, layout, vis, nbuf), nbuf)


def forced(cfg):
    """(vis or None, nbuf) that MINIGRID_B200_CFG="warps,vis,nbuf" forces."""
    c = [int(v) for v in cfg.split(",")] if cfg else [0, 0, 0]
    return (c[1] or None), (2 if c[2] == 2 else 1)


def plan_vis_nbuf(spec, layout, cfg):
    vis, nbuf = forced(cfg)
    return (VIS_NONE if spec.see_through_walls else (vis or VIS_TBL)), (1 if layout == WINDOW else nbuf)


def predicted_smem(env_id, cfg):
    """The plan configure_step prefers: the warp count nearest its target (22 one-buffer, 14 two-buffer, 20 window)."""
    s = ALL_IDS[env_id]
    layout = layout_of(s)
    vis, nbuf = plan_vis_nbuf(s, layout, cfg)
    target = 20 if layout == WINDOW else (14 if nbuf == 2 else 22)
    return step_smem_bytes(s.width, s.height, layout, vis, min(target, search_warps(s.width, s.height, layout, vis, nbuf)), nbuf)


KIND_NAMES = {v: k[5:].lower() for k, v in vars(specs).items() if k.startswith("KIND_")}


def k1_groups(cfg=None):
    """The registered ids grouped by K1 kernel (kind, see-through, layout), one id per geometry (the first registered;
    MiniGrid ids before BabyAI ones), largest predicted plan first. Only groups with two or more geometries."""
    groups = {}
    for env_id, s in ALL_IDS.items():
        layout = layout_of(s)
        name = f"{KIND_NAMES[s.kind]}-{'see' if s.see_through_walls else 'vis'}-{'window' if layout else 'tiled'}"
        groups.setdefault(name, {}).setdefault((s.width, s.height), env_id)
    return {name: sorted(g.values(), key=lambda i: -predicted_smem(i, cfg)) for name, g in groups.items() if len(g) > 1}


# the groups in which the handle created last would have left a limit below the first handle's plan.smem
ADVERSARIAL = {
    None: {"doorkey-vis-tiled": False, "crossing-vis-tiled": False, "lavagap-vis-tiled": False, "redbluedoors-vis-tiled": True,
           "memory-vis-tiled": True, "dynobs-see-tiled": True, "roomgrid-vis-tiled": True, "roomgrid-vis-window": False,
           "empty-see-tiled": False, "gotodoor-see-tiled": False, "fetch-see-tiled": False, "gotoobject-see-tiled": False,
           "putnear-see-tiled": False},
    "0,0,2": {"roomgrid-vis-tiled": True},
    "0,1,0": {"roomgrid-vis-tiled": True},
}


def sweep_cases():
    cases = []
    for i, name in enumerate(sorted(k1_groups())):
        both = name.startswith(("roomgrid", "dynobs"))
        for mode in (("next_step", "same_step") if both else (("next_step", "same_step")[i % 2],)):
            cases.append(pytest.param(name, mode, None, id=f"{name}-{mode}"))
    cases.append(pytest.param("roomgrid-vis-tiled", "next_step", "0,0,2", id="roomgrid-vis-tiled-next_step-two-buffer"))
    cases.append(pytest.param("roomgrid-vis-tiled", "same_step", "0,1,0", id="roomgrid-vis-tiled-same_step-alu"))
    return cases


# ---- handles, plans and oracles ----
def create(case, env_id, n, mode, monkeypatch, capfd, cfg=None):
    """MinigridVecEnv with its K1 plan line, checked against the mirror: layout, forced options and smem."""
    if cfg:
        monkeypatch.setenv("MINIGRID_B200_CFG", cfg)
    capfd.readouterr()
    env = MinigridVecEnv(env_id, n, autoreset_mode=mode)
    monkeypatch.delenv("MINIGRID_B200_CFG", raising=False)
    plans = PLAN_RE.findall(capfd.readouterr().err)
    assert plans, "MINIGRID_B200_VERBOSE=1 printed no K1 plan line"
    plan = dict(zip(("layout", "warps", "vis", "nbuf", "ctas", "grid", "smem", "tiles"), map(int, plans[-1])))
    s = ALL_IDS[env_id]
    layout = layout_of(s)
    vis, nbuf = plan_vis_nbuf(s, layout, cfg)
    assert (plan["layout"], plan["vis"], plan["nbuf"]) == (layout, vis, nbuf), f"{case}: {env_id}: K1 plan {plan}"
    mirror = step_smem_bytes(s.width, s.height, layout, plan["vis"], plan["warps"], plan["nbuf"])
    assert plan["smem"] == mirror, f"{case}: {env_id}: plan smem {plan['smem']} B, the mirror of step_smem_bytes {mirror} B"
    assert plan["warps"] <= search_warps(s.width, s.height, layout, plan["vis"], plan["nbuf"]), f"{case}: {env_id}: {plan}"
    return env, plan


def make_oracle(env_id, n, mode, hashed=False):
    if env_id in specs.BABYAI_PICKUP_PUTNEXT_REGISTRY:
        return PickupOracle(env_id, n, autoreset=mode, n_threads=0)
    if env_id in specs.BABYAI_REGISTRY:
        return BabyAIOracle(env_id, n, autoreset=mode, n_threads=0)
    if hashed:
        return hs.HashedOracle(env_id, n, autoreset=mode)
    return OracleVecEnv(None, n, spec=hs.oracle_spec(env_id), autoreset=mode, n_threads=0)


def assert_adversarial(case, first_id, first_plan, later_id, expected):
    """Whether the old rule's limit after `later_id`'s mg_create is below the first handle's plan.smem."""
    s = ALL_IDS[later_id]
    left = old_limit(s, layout_of(s), first_plan["vis"], first_plan["nbuf"])
    assert (left < first_plan["smem"]) == expected, \
        (f"{case}: {later_id} would have left a limit of {left} B for {first_id}'s plan of {first_plan['smem']} B: "
         f"expected this case {'' if expected else 'not '}to be adversarial")


def ends_before_last(ends):
    return int(sum(ends[:-1]))


# ---- 1. every K1 kernel that several geometries share ----
@pytest.mark.parametrize("group,mode,cfg", sweep_cases())
def test_group_sweep(group, mode, cfg, monkeypatch, capfd):
    """One handle per geometry of the group, the largest plan created first, then all stepped interleaved for 40 steps
    with injected sparse ends and a whole-tile wave. Afterwards the first handle's full_obs, and its hash() on a sample
    (MiniGrid ids), against the oracle."""
    case = f"sweep/{group}/{mode}/{cfg or 'default'}"
    ids = k1_groups(cfg)[group]
    n, T = 2085, 40
    envs, orcs, plans, acts = [], [], [], []
    for k, env_id in enumerate(ids):
        env, plan = create(case, env_id, n, mode, monkeypatch, capfd, cfg)
        orc = make_oracle(env_id, n, mode, hashed=k == 0)
        env.reset(seed=2000 + k)
        orc.reset(seed=2000 + k)
        inject_ends(env, orc, n, min(T - 4, env.max_steps), (3, 40), 8, seed=20 + k)
        envs.append(env)
        orcs.append(orc)
        plans.append(plan)
        acts.append(random_actions(T, n, seed=40 + k)[1])
    assert plans[0]["smem"] == max(p["smem"] for p in plans), \
        f"{case}: {ids[0]} was created first, but {[p['smem'] for p in plans]} are the plans' smem"
    assert_adversarial(case, ids[0], plans[0], ids[-1], ADVERSARIAL[cfg][group])
    ends = [[] for _ in ids]
    for t in range(T):
        for k, env in enumerate(envs):
            a = acts[k][t]
            env.step(torch.as_tensor(a, device="cuda"))
            o = orcs[k].step(a)
            check_outputs(f"{case}: {ids[k]}", f"step {t}", engine_outputs(env), o)
            ends[k].append(int((np.asarray(o[3], bool) | np.asarray(o[4], bool)).sum()))
        if t % 10 == 9:
            for k, env in enumerate(envs):
                check_state(f"{case}: {ids[k]}", f"after step {t}", env, orcs[k])
    for k in range(len(ids)):
        assert ends_before_last(ends[k]) > 0, f"{case}: {ids[k]}: no episode ended inside the run"
    first, orc = envs[0], orcs[0]
    first_diff(case, f"{ids[0]} full_obs", "full_obs", first.full_obs().cpu().numpy(), getattr(orc, "o", orc).full_obs())
    if isinstance(orc, hs.HashedOracle):
        sample = np.concatenate([np.arange(32), np.arange((n - 1) // 32 * 32, n)])  # the first and the (ragged) last tile
        got = first.hash(64)
        for i, h in zip(sample, orc.hash(64, envs=sample)):
            assert got[i] == h, f"{case}: {ids[0]}: hash of env {i} (tile {i // 32})"
    for env in envs:
        env.close()


# ---- 2. a captured graph across an mg_create ----
def test_graph_replay_across_create(monkeypatch, capfd):
    """8 public step() calls of KeyCorridorS4R3 captured as bench.py captures them; then a KeyCorridorS3R1 handle (the
    same K1 kernel, a smaller tile) is created, stepped and destroyed; then the graph is replayed twice with fresh
    actions and the handle stepped eagerly once more."""
    big, small = "MiniGrid-KeyCorridorS4R3-v0", "MiniGrid-KeyCorridorS3R1-v0"
    case, n, G, W, replays = "graph-across-create", 2085, 8, 3, 2
    env, plan = create(case, big, n, "next_step", monkeypatch, capfd)
    orc = make_oracle(big, n, "next_step")
    env.reset(seed=3000)
    orc.reset(seed=3000)
    inject_ends(env, orc, n, W + (replays + 1) * G, (5, 40), W + G + 2, seed=30)
    table, table_np = random_actions(G, n, seed=31)
    rows = [table[i] for i in range(G)]
    fresh, fresh_np = random_actions(replays * G + 1, n, seed=32)
    for t in range(W):
        env.step(rows[t])
        check_outputs(case, f"eager step {t}", engine_outputs(env), orc.step(table_np[t]))
    cap = torch.cuda.Stream()
    cap.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cap):
        for t in range(G):
            env.step(rows[t])
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=cap):
            for t in range(G):
                env.step(rows[t])
    torch.cuda.current_stream().wait_stream(cap)
    torch.cuda.synchronize()
    for t in range(G):
        o = orc.step(table_np[t])
    check_outputs(case, "after the warm-up", engine_outputs(env), o)

    other, _ = create(case, small, n, "next_step", monkeypatch, capfd)
    assert_adversarial(case, big, plan, small, True)
    other.reset(seed=1)
    other.step(torch.zeros(n, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    other.close()
    del other

    ends = 0
    for r in range(replays):
        table.copy_(fresh[r * G:(r + 1) * G])
        launches = env.launch_count
        graph.replay()
        torch.cuda.synchronize()
        assert env.launch_count == launches, f"{case}: the C-ABI was called during replay {r}"
        for t in range(G):
            o = orc.step(fresh_np[r * G + t])
            ends += int((np.asarray(o[3], bool) | np.asarray(o[4], bool)).sum())
        check_outputs(case, f"last step of replay {r}", engine_outputs(env), o)
        check_state(case, f"after replay {r}", env, orc)
    assert ends > 0, f"{case}: no episode ended inside the replays"
    env.step(fresh[replays * G])
    check_outputs(case, "eager step after the replays", engine_outputs(env), orc.step(fresh_np[replays * G]))
    check_state(case, "at the end", env, orc)


# ---- 3. handles created and destroyed around a long-lived one ----
CYCLE_IDS = ("MiniGrid-MemoryS7-v0", "MiniGrid-DoorKey-5x5-v0", "MiniGrid-MemoryS13-v0", "MiniGrid-FourRooms-v0",
             "MiniGrid-Dynamic-Obstacles-16x16-v0", "BabyAI-GoToLocalS6N2-v0", "MiniGrid-MemoryS11-v0",
             "MiniGrid-Empty-5x5-v0", "MiniGrid-KeyCorridorS3R1-v0", "MiniGrid-MemoryS17Random-v0")
# MemoryS9's kernel: whether each of these would have left a limit below MemoryS9's plan
MEMORY_ADVERSARIAL = {"MiniGrid-MemoryS7-v0": True, "MiniGrid-MemoryS13-v0": True, "MiniGrid-MemoryS11-v0": False}
MEM_TOL = 1 << 30  # other work on the device may hold memory for a while; 30 leaked handles would hold far more


def free_device_bytes():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_create_destroy_cycles(monkeypatch, capfd):
    """30 handles of varied ids and kinds (three in ten of MemoryS9's K1 kernel), each created, reset, stepped and
    closed twice, while a MemoryS9 handle takes one step against the oracle per cycle. Afterwards the device's free
    memory is back at its baseline within MEM_TOL."""
    case, n, N, cycles = "create-destroy", 2085, 1 << 19, 30
    env, plan = create(case, "MiniGrid-MemoryS9-v0", n, "same_step", monkeypatch, capfd)
    orc = make_oracle("MiniGrid-MemoryS9-v0", n, "same_step")
    env.reset(seed=4000)
    orc.reset(seed=4000)
    inject_ends(env, orc, n, cycles - 4, (3, 40), 6, seed=41)
    _, a_np = random_actions(cycles, n, seed=42)
    base = free_device_bytes()
    held, ends = 0, 0
    for c in range(cycles):
        env_id = CYCLE_IDS[c % len(CYCLE_IDS)]
        before = free_device_bytes()
        other = MinigridVecEnv(env_id, N, autoreset_mode=("next_step", "same_step")[c % 2])
        if env_id in MEMORY_ADVERSARIAL:
            assert_adversarial(case, "MiniGrid-MemoryS9-v0", plan, env_id, MEMORY_ADVERSARIAL[env_id])
        other.reset(seed=c)
        other.step(torch.full((N,), c % 7, dtype=torch.int32, device="cuda"))
        held += before - free_device_bytes()
        env.step(torch.as_tensor(a_np[c], device="cuda"))
        o = orc.step(a_np[c])
        check_outputs(case, f"cycle {c} ({env_id} alive)", engine_outputs(env), o)
        ends += int((np.asarray(o[3], bool) | np.asarray(o[4], bool)).sum())
        other.close()
        other.close()
        del other
    check_state(case, f"after {cycles} cycles", env, orc)
    assert ends > 0, f"{case}: no episode of the long-lived handle ended"
    assert held > 4 * MEM_TOL, f"{case}: the cycled handles held {held} B in all: too little to show a leak"
    drop = base - free_device_bytes()
    for _ in range(10):  # memory another process holds for a moment is not a leak
        if drop <= MEM_TOL:
            break
        time.sleep(0.5)
        drop = base - free_device_bytes()
    assert drop <= MEM_TOL, f"{case}: {drop} B of device memory not returned after {cycles} handles were destroyed"


# ---- 4. the process-wide host expansion pool ----
def test_host_pool_two_threads(monkeypatch, capfd):
    """Two packed-format handles of one K1 kernel (KeyCorridorS4R3, then KeyCorridorS3R1) with different pool thread
    counts, each driven through step_host by its own Python thread at the same time; every step's host outputs against
    the oracle afterwards."""
    case, n, T = "host-pool", 33000, 16
    pairs = (("MiniGrid-KeyCorridorS4R3-v0", 2), ("MiniGrid-KeyCorridorS3R1-v0", 5))
    envs, orcs, plans, acts = [], [], [], []
    for k, (env_id, threads) in enumerate(pairs):
        env, plan = create(case, env_id, n, "next_step", monkeypatch, capfd)
        env.set_host_format("packed", threads)
        assert env.host_threads == threads
        orc = make_oracle(env_id, n, "next_step")
        obs, _ = env.reset_host(seed=5000 + k)
        first_diff(f"{case}: {env_id}", "reset_host", "obs", obs["image"].numpy(), orc.reset(seed=5000 + k)[0])
        inject_ends(env, orc, n, T - 4, (3, 400), 6, seed=50 + k)
        plans.append(plan)
        envs.append(env)
        orcs.append(orc)
        acts.append(random_actions(T, n, seed=51 + k)[1])
    assert_adversarial(case, pairs[0][0], plans[0], pairs[1][0], True)
    got, errors = [[], []], []
    start = threading.Barrier(2)

    def drive(k):
        try:
            start.wait()
            for t in range(T):
                obs, r, te, tr, _ = envs[k].step_host(acts[k][t])
                got[k].append(tuple(x.numpy().copy() for x in (obs["image"], obs["direction"], r, te, tr)))
        except BaseException as e:  # noqa: BLE001 (re-raised in the main thread)
            errors.append(e)

    workers = [threading.Thread(target=drive, args=(k,)) for k in range(2)]
    for w in workers:
        w.start()
    for w in workers:
        w.join()
    if errors:
        raise errors[0]
    for k, (env_id, _) in enumerate(pairs):
        ends = 0
        for t in range(T):
            o = orcs[k].step(acts[k][t])
            check_outputs(f"{case}: {env_id}", f"step {t}", got[k][t], o)
            ends += int((np.asarray(o[3], bool) | np.asarray(o[4], bool)).sum())
        check_state(f"{case}: {env_id}", f"after {T} steps", envs[k], orcs[k])
        assert ends > 0, f"{case}: {env_id}: no episode ended"
