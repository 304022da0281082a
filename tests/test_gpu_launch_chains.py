"""K1 (mg_step: transition + autoreset + observation) launched the way the benchmark and a training loop launch it, bit for
bit against the oracle: back-to-back chains with no host synchronisation between steps (programmatic dependent launch:
the next step's prologue runs while the previous grid drains), CUDA-graph replays, observation buffers at every address
residue mod 16 (full tiles go through the bulk store only when the pointer is 16-byte aligned, else through the byte
copy), more tiles per CTA than K1's order list holds, handles stepped on two streams at once, and consumer kernels
between steps. Each step writes into its own slot of a guarded allocation, so that a write outside the slot shows up as
an overwritten canary byte. Every case also checks the K1 plan line (MINIGRID_B200_VERBOSE) to prove which kernel ran."""
import os
import re

import numpy as np
import pytest
import torch

import hash_support as hs
from babyai_oracle import BabyAIOracle
from minigrid_b200 import MinigridVecEnv, _lib, specs
from oracle.oracle import OracleVecEnv

pytestmark = pytest.mark.gpu

FIELDS = ("obs", "dir", "reward", "terminated", "truncated")
CANARY = 0xA5
OBS_RESIDUES = (0, 1, 5, 8, 15)  # obs slot addresses mod 16: aligned (bulk store) and unaligned (byte copy) alternate
TILED, WINDOW = 0, 1
PLAN_RE = re.compile(r"K1 plan: layout=(\d+), (\d+) warps/CTA, vis=(\d+), nbuf=(\d+), (\d+) CTA/SM, grid=(\d+), smem=\d+ B, "
                     r"tiles=(\d+)")
DENSE_RESET_MIN = 8  # warp_reset's threshold for the whole-tile (dense) reset path, mg_step_kernel.cuh


@pytest.fixture(autouse=True)
def _launch_knobs(monkeypatch):
    # MINIGRID_B200_PDL is read once per process: these tests are about the default launch (PDL on) and cannot toggle it
    assert "MINIGRID_B200_PDL" not in os.environ, "unset MINIGRID_B200_PDL: the chains test the programmatic dependent launch"
    for knob in ("MINIGRID_B200_CFG", "MINIGRID_B200_GRID", "MINIGRID_B200_LAYOUT", "MINIGRID_B200_HOTFIRST"):
        monkeypatch.delenv(knob, raising=False)
    monkeypatch.setenv("MINIGRID_B200_VERBOSE", "1")


# ---- guarded output slots ----
class Guarded:
    """`n_slots` slots of `slot_bytes` each in one device allocation filled with CANARY: at least GAP canary bytes before
    the first slot, between slots and after the last. Slot t starts at an address = residues[t % len] (mod 16)."""
    GAP = 40

    def __init__(self, n_slots, slot_bytes, residues):
        self.size = slot_bytes
        self.starts = []
        pos = 0
        for t in range(n_slots):
            pos = (pos + self.GAP + 15) // 16 * 16 + residues[t % len(residues)]
            self.starts.append(pos)
            pos += slot_bytes
        self.total = pos + self.GAP
        self.buf = torch.full((self.total,), CANARY, dtype=torch.uint8, device="cuda")
        assert self.buf.data_ptr() % 16 == 0
        self.host = None

    def ptr(self, t):
        return self.buf.data_ptr() + self.starts[t]

    def tensor(self, t):
        return self.buf[self.starts[t]:self.starts[t] + self.size]

    def fetch(self):
        self.host = self.buf.cpu().numpy()

    def slot(self, t, dtype):
        s = self.starts[t]
        return np.frombuffer(self.host[s:s + self.size].tobytes(), dtype)

    def check_canaries(self, what):
        inside = np.zeros(self.total, bool)
        for s in self.starts:
            inside[s:s + self.size] = True
        bad = np.nonzero(~inside & (self.host != CANARY))[0]
        if bad.size:
            b = int(bad[0])
            k = int(np.searchsorted(self.starts, b, side="right")) - 1
            where = "before slot 0" if k < 0 else f"{b - self.starts[k] - self.size} bytes past the end of slot {k}"
            raise AssertionError(f"{what}: {bad.size} canary bytes overwritten, the first {where} (0x{self.host[b]:02x})")

    def residues(self):
        return {self.ptr(t) % 16 for t in range(len(self.starts))}


class Slots:
    """Per-step output slots of mg_step, one guarded allocation per output."""
    LAYOUT = {"obs": (147, np.uint8, OBS_RESIDUES), "dir": (4, np.int32, (0, 4, 8, 12)), "reward": (8, np.float64, (0, 8)),
              "terminated": (1, np.uint8, (0, 3, 7, 9, 14)), "truncated": (1, np.uint8, (2, 6, 11, 13, 15))}

    def __init__(self, T, n):
        self.n = n
        self.g = {k: Guarded(T, n * per, res) for k, (per, _, res) in self.LAYOUT.items()}

    def ptrs(self, t):
        return [self.g[k].ptr(t) for k in FIELDS]

    def fetch(self):
        for g in self.g.values():
            g.fetch()

    def outputs(self, t):
        out = [self.g[k].slot(t, self.LAYOUT[k][1]) for k in FIELDS]
        out[0] = out[0].reshape(self.n, 7, 7, 3)
        return out

    def check_canaries(self, case):
        for k in FIELDS:
            self.g[k].check_canaries(f"{case}: {k} slots")

    def assert_mixed_alignment(self, case):
        r = self.g["obs"].residues()
        assert 0 in r and len(r) > 1, f"{case}: obs slots at residues {sorted(r)}: the chain must mix aligned and unaligned"


# ---- engines, oracles, comparisons ----
def stream():
    return torch.cuda.current_stream().cuda_stream


def step_into(env, actions_row, slots, t):
    """One mg_step of `env` on the current stream into slot t: the C-ABI call itself, nothing else enqueued."""
    _lib.check(_lib.load().mg_step(env._h, actions_row.data_ptr(), 0, *slots.ptrs(t), stream()))


def make_engine(env_id, n, mode, monkeypatch, capfd, cfg=None, grid=None):
    if cfg:
        monkeypatch.setenv("MINIGRID_B200_CFG", cfg)
    if grid:
        monkeypatch.setenv("MINIGRID_B200_GRID", str(grid))
    capfd.readouterr()
    env = MinigridVecEnv(env_id, n, autoreset_mode=mode)
    plans = PLAN_RE.findall(capfd.readouterr().err)
    assert plans, "MINIGRID_B200_VERBOSE=1 printed no K1 plan line"
    k = dict(zip(("layout", "warps", "vis", "nbuf", "ctas", "grid", "tiles"), map(int, plans[-1])))
    monkeypatch.delenv("MINIGRID_B200_CFG", raising=False)
    monkeypatch.delenv("MINIGRID_B200_GRID", raising=False)
    return env, k


def check_plan(case, plan, env_id, n, layout, cfg=None, grid=None):
    """The plan mg_create chose: layout, buffers per warp, visibility form, grid and tile count."""
    c = [int(v) for v in cfg.split(",")] if cfg else [0, 0, 0]
    want = {"layout": layout, "tiles": (n + 31) // 32,
            "vis": 0 if specs.get(env_id).see_through_walls else (1 if c[1] == 1 else 2),
            "nbuf": 2 if c[2] == 2 else 1}
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    want["grid"] = int(grid) if grid else min(sms * plan["ctas"], (want["tiles"] + plan["warps"] - 1) // plan["warps"])
    got = {k: plan[k] for k in want}
    assert got == want, f"{case}: K1 plan {plan}, expected {want}"


def assert_order_list_live(case, plan, mode):
    """NEXT_STEP with more tiles per CTA than warps: every CTA orders its tiles through K1's order list (flagged tiles
    first, the others in the direction the launch parity picks), built before griddepcontrol.wait."""
    if mode == "next_step":
        per_cta = plan["tiles"] // plan["grid"]
        assert per_cta > plan["warps"], \
            f"{case}: {per_cta} tiles per CTA for {plan['warps']} warps: K1's order list is not in use"


def make_oracle(env_id, n, mode):
    if env_id.startswith("BabyAI"):
        return BabyAIOracle(env_id, n, autoreset=mode, n_threads=0)
    return OracleVecEnv(env_id, n, autoreset=mode, n_threads=0)


def set_agents(env, orc, agent):
    env.set_state(agent=agent)
    getattr(orc, "c", orc).set_state(agent=agent)  # BabyAIOracle: the C oracle underneath holds the records


def inject_ends(env, orc, n, span, wave_tiles, wave_k, seed):
    """The same step counts on both sides: about half the envs truncate at a random step in [0, span - 1) of what
    follows (sparse ends), and every env of `wave_tiles` at step wave_k - 1 (a whole-tile wave)."""
    rng = np.random.default_rng(seed)
    agent = orc.get_state()["agent"].copy()
    sparse = rng.random(n) < 0.5
    agent[sparse, 5] = env.max_steps - rng.integers(1, span, int(sparse.sum()))
    for tile in wave_tiles:
        agent[tile * 32:(tile + 1) * 32, 5] = env.max_steps - wave_k
    set_agents(env, orc, agent)


def first_diff(case, where, name, x, y, envs=None):
    n = y.shape[0]
    diff = (x.reshape(n, -1) != y.reshape(n, -1)).any(axis=1)
    if diff.any():
        i = int(np.argmax(diff))
        e = i if envs is None else int(envs[i])
        xr, yr = x.reshape(n, -1)[i], y.reshape(n, -1)[i]
        j = int(np.argmax(xr != yr))
        raise AssertionError(f"{case}: {where}: {name} differs in {int(diff.sum())} envs, the first env {e} (tile {e // 32}) "
                             f"from element {j} of {xr.size}: engine {xr[j:j + 12].tolist()} oracle {yr[j:j + 12].tolist()}")


def check_outputs(case, where, got, want, envs=None):
    for name, x, y in zip(FIELDS, got, want):
        x, y = np.asarray(x), np.asarray(y)
        if name == "reward":  # IEEE bit patterns
            x, y = np.ascontiguousarray(x, np.float64).view(np.uint64), np.ascontiguousarray(y, np.float64).view(np.uint64)
        elif name in ("terminated", "truncated"):
            x, y = x.astype(np.uint8), y.astype(np.uint8)
        else:
            y = y.astype(x.dtype)
        first_diff(case, where, name, x, y, envs)


def engine_state(env):
    st = {k: v.cpu().numpy() for k, v in env.get_state().items()}
    st["rng"] = st["rng"].view(np.uint64)
    return st


def check_state(case, where, env, orc, envs=None):
    es, os_ = engine_state(env), orc.get_state()
    for k in ("grid", "agent", "rng", "pending"):
        x = es[k] if envs is None else es[k][envs]
        first_diff(case, where, k, x, np.asarray(os_[k]).astype(x.dtype), envs)


def engine_outputs(env):
    """What the last step() left in the handle's reused buffers."""
    return (env._image.cpu().numpy(), env._direction.cpu().numpy(), env._reward.cpu().numpy(),
            env._terminated.cpu().numpy(), env._truncated.cpu().numpy())


def copy_outputs(o):
    return tuple(np.array(x, copy=True) for x in o)


def random_actions(T, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    acts = torch.randint(0, 7, (T, n), generator=g, device="cuda", dtype=torch.int32)
    return acts, acts.cpu().numpy()


def run_chain_and_compare(case, env, orc, acts, a_np, T, slots):
    """T back-to-back steps into their own slots, ONE synchronisation at the end, then every step against the oracle.
    Returns the oracle's per-step outputs."""
    for t in range(T):
        step_into(env, acts[t], slots, t)
    torch.cuda.synchronize()
    slots.fetch()
    want = []
    for t in range(T):
        o = copy_outputs(orc.step(a_np[t]))
        check_outputs(case, f"step {t}", slots.outputs(t), o)
        want.append(o)
    check_state(case, f"after {T} steps", env, orc)
    slots.check_canaries(case)
    slots.assert_mixed_alignment(case)
    return want


def ends_per_tile(o, n):
    """Episode ends (terminated | truncated) per tile of one step's outputs."""
    done = (np.asarray(o[3], bool) | np.asarray(o[4], bool)).astype(np.int64)
    return np.bincount(np.arange(n) // 32, weights=done, minlength=(n + 31) // 32)


def assert_resets_inside(case, want, n, wave_step):
    """Episodes ended before the chain's last step (so their autoresets ran inside it), sparse ones (a few envs of a tile)
    and a dense one (>= DENSE_RESET_MIN envs of a tile at once)."""
    per = np.stack([ends_per_tile(o, n) for o in want[:-1]])
    assert per.sum() > 0, f"{case}: no episode ended inside the chain"
    assert ((per > 0) & (per < DENSE_RESET_MIN)).any(), f"{case}: no sparse ends inside the chain"
    assert per[wave_step].max() >= DENSE_RESET_MIN, f"{case}: no whole-tile wave at step {wave_step}"


# ---- 1. eager chains ----
EAGER = [  # case, env_id, expected layout, MINIGRID_B200_CFG, reward wrappers, n
    ("doorkey", "MiniGrid-DoorKey-8x8-v0", TILED, None, None, 4133),
    ("doorkey-tiled2", "MiniGrid-DoorKey-8x8-v0", TILED, "0,0,2", None, 4133),
    ("doorkey-alu", "MiniGrid-DoorKey-8x8-v0", TILED, "0,1,0", None, 4133),
    ("fourrooms", "MiniGrid-FourRooms-v0", WINDOW, None, None, 4133),
    ("obstructedmaze-full-v1", "MiniGrid-ObstructedMaze-Full-v1", WINDOW, None, None, 4133),
    ("dynobs", "MiniGrid-Dynamic-Obstacles-8x8-v0", TILED, None, None, 4133),
    ("fetch", "MiniGrid-Fetch-8x8-N3-v0", TILED, None, None, 4133),
    ("lavacrossing-nodeath-bonus", "MiniGrid-LavaCrossingS9N1-v0", TILED, None, (("lava",), "action"), 4133),
    ("babyai-gotolocal", "BabyAI-GoToLocal-v0", TILED, None, None, 2085),
]


@pytest.mark.parametrize("grid", [None, 2], ids=["grid-default", "grid-2"])
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
@pytest.mark.parametrize("case,env_id,layout,cfg,wrap,n", EAGER, ids=[c[0] for c in EAGER])
def test_eager_chain(case, env_id, layout, cfg, wrap, n, mode, grid, monkeypatch, capfd):
    """48 back-to-back steps with sparse ends and a whole-tile wave inside the chain. The next grid's CTAs find idle
    SMs and run their prologue while the previous grid drains. With two CTAs (grid-2) in NEXT_STEP mode every CTA has
    more tiles than warps, so that prologue builds the CTA's tile order from flags the previous grid may still be
    writing."""
    case = f"{case}/{mode}/grid={grid or 'default'}"
    T = 48
    env, plan = make_engine(env_id, n, mode, monkeypatch, capfd, cfg=cfg, grid=grid)
    check_plan(case, plan, env_id, n, layout, cfg, grid)
    if grid:
        assert_order_list_live(case, plan, mode)
    orc = make_oracle(env_id, n, mode)
    if wrap:
        for e in (env, orc):
            e.set_no_death(wrap[0], -1.25)
            e.set_bonus(wrap[1])
    env.reset(seed=600)
    orc.reset(seed=600)
    tiles = (n + 31) // 32
    wave_k = 12
    inject_ends(env, orc, n, T - 4, (0, tiles // 2, tiles - 1), wave_k, seed=1)
    acts, a_np = random_actions(T, n, seed=2)
    slots = Slots(T, n)
    want = run_chain_and_compare(case, env, orc, acts, a_np, T, slots)
    assert_resets_inside(case, want, n, wave_k - 1)


# ---- 2. CUDA-graph chains ----
@pytest.mark.parametrize("G", [16, 15])
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
@pytest.mark.parametrize("env_id,layout", [("MiniGrid-DoorKey-8x8-v0", TILED), ("MiniGrid-FourRooms-v0", WINDOW),
                                           ("MiniGrid-Dynamic-Obstacles-8x8-v0", TILED)])
def test_graph_chain_c_abi(env_id, layout, mode, G, monkeypatch, capfd):
    """G per-slot mg_step calls captured on a side stream (after warming it, as bench.py does) and replayed 4 times
    with fresh actions copied into the captured rows; a whole-tile wave ends inside the first replay. Two CTAs: in
    NEXT_STEP mode the order list is in use, and with an odd G the order direction frozen into each captured launch
    no longer alternates from the last step of one replay to the first step of the next."""
    case = f"graph-c-abi/{env_id}/{mode}/G={G}"
    n, replays = 4133, 4
    env, plan = make_engine(env_id, n, mode, monkeypatch, capfd, grid=2)
    check_plan(case, plan, env_id, n, layout, grid=2)
    assert_order_list_live(case, plan, mode)
    orc = make_oracle(env_id, n, mode)
    env.reset(seed=700)
    orc.reset(seed=700)
    wave_k = G + 3  # step G + 2: the third step of the first replay
    inject_ends(env, orc, n, (replays + 1) * G, (5, 40, 70, 100), wave_k, seed=3)
    rows = torch.empty((G, n), dtype=torch.int32, device="cuda")  # the captured action rows
    fresh, fresh_np = random_actions((replays + 1) * G, n, seed=4)
    slots = Slots(G, n)
    cap = torch.cuda.Stream()
    rows.copy_(fresh[:G])
    cap.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cap):
        for t in range(G):  # warm the capture stream: real steps
            step_into(env, rows[t], slots, t)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=cap):
            for t in range(G):
                step_into(env, rows[t], slots, t)
    torch.cuda.current_stream().wait_stream(cap)
    torch.cuda.synchronize()
    slots.fetch()
    want = []
    for t in range(G):
        want.append(copy_outputs(orc.step(fresh_np[t])))
        check_outputs(case, f"warm-up step {t}", slots.outputs(t), want[-1])
    for r in range(1, replays + 1):
        rows.copy_(fresh[r * G:(r + 1) * G])
        launches = env.launch_count
        graph.replay()
        torch.cuda.synchronize()
        assert env.launch_count == launches, f"{case}: the C-ABI was called during replay {r}"
        slots.fetch()
        for t in range(G):
            o = copy_outputs(orc.step(fresh_np[r * G + t]))
            check_outputs(case, f"replay {r} step {t}", slots.outputs(t), o)
            want.append(o)
        check_state(case, f"after replay {r}", env, orc)
        slots.check_canaries(f"{case} replay {r}")
    slots.assert_mixed_alignment(case)
    assert_resets_inside(case, want, n, wave_k - 1)


def mini_bench(case, envs, act_rows, T, W, G, K):
    """bench.py's loop: W eager steps, G eager steps on the capture stream, a G-step graph and a remainder graph of the
    public step() calls of R rotating batches, one warm replay, then K steps of replays. Returns, per batch, the action
    rows its executed steps used, in order, and the launch counts before the replays."""
    R = len(envs)
    rows_run = [[] for _ in range(R)]

    def eager_run(steps, first=0, record=True):
        for t in range(first, first + steps):
            envs[t % R].step(act_rows[t % T])
            if record:
                rows_run[t % R].append(t % T)

    def replay(g, first, steps):
        g.replay()
        for t in range(first, first + steps):
            rows_run[t % R].append(t % T)

    eager_run(W)
    torch.cuda.synchronize()
    rem = K % G
    cap = torch.cuda.Stream()
    cap.wait_stream(torch.cuda.current_stream())
    graph_rem = None
    with torch.cuda.stream(cap):
        eager_run(G)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=cap):
            eager_run(G, record=False)
        if rem:
            graph_rem = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph_rem, stream=cap):
                eager_run(rem, G * (K // G), record=False)
    torch.cuda.current_stream().wait_stream(cap)
    torch.cuda.synchronize()
    launches = [e.launch_count for e in envs]
    replay(graph, 0, G)
    for _ in range(K // G):
        replay(graph, 0, G)
    if rem:
        replay(graph_rem, G * (K // G), rem)
    torch.cuda.synchronize()
    for b, e in enumerate(envs):
        assert e.launch_count == launches[b], f"{case}: batch {b}: the C-ABI was called during the replays"
    return rows_run


@pytest.mark.parametrize("G", [16, 15])
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
@pytest.mark.parametrize("env_id,layout", [("MiniGrid-DoorKey-8x8-v0", TILED), ("MiniGrid-FourRooms-v0", WINDOW),
                                           ("MiniGrid-Dynamic-Obstacles-8x8-v0", TILED)])
def test_graph_chain_public_step(env_id, layout, mode, G, monkeypatch, capfd):
    """MinigridVecEnv.step with its reused buffers captured as bench.py captures it, replayed 4 times with fresh
    actions copied into the table; the state and the last step's outputs after each replay. Two CTAs, as in
    test_graph_chain_c_abi: the order list is in use in NEXT_STEP mode."""
    case = f"graph-step/{env_id}/{mode}/G={G}"
    n, replays, W = 4133, 4, 3
    env, plan = make_engine(env_id, n, mode, monkeypatch, capfd, grid=2)
    check_plan(case, plan, env_id, n, layout, grid=2)
    assert_order_list_live(case, plan, mode)
    orc = make_oracle(env_id, n, mode)
    env.reset(seed=800)
    orc.reset(seed=800)
    wave_k = W + G + 3  # the third step of the first replay
    inject_ends(env, orc, n, W + (replays + 2) * G, (9, 40, 70, 100), wave_k, seed=5)
    table, table_np = random_actions(G, n, seed=6)
    rows = [table[i] for i in range(G)]
    fresh, fresh_np = random_actions(replays * G, n, seed=7)
    want = []
    for t in range(W):
        env.step(rows[t])
        want.append(copy_outputs(orc.step(table_np[t])))
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
        want.append(copy_outputs(orc.step(table_np[t])))
    check_outputs(case, "after the warm-up", engine_outputs(env), want[-1])
    for r in range(replays):
        table.copy_(fresh[r * G:(r + 1) * G])
        launches = env.launch_count
        graph.replay()
        torch.cuda.synchronize()
        assert env.launch_count == launches, f"{case}: the C-ABI was called during replay {r}"
        for t in range(G):
            want.append(copy_outputs(orc.step(fresh_np[r * G + t])))
        check_outputs(case, f"last step of replay {r}", engine_outputs(env), want[-1])
        check_state(case, f"after replay {r}", env, orc)
    assert_resets_inside(case, want, n, wave_k - 1)


# ---- 3. a miniature of the benchmark ----
def desync_both(env, orc, seed, envs=None):
    """bench.py's desync: step_count ~ U[0, max_steps), the same draw on both sides (`envs`: the oracle holds a sample)."""
    draw = np.random.default_rng(seed).integers(0, env.max_steps, env.num_envs).astype(np.int32)
    agent = engine_state(env)["agent"]
    agent[:, 5] = draw
    env.set_state(agent=agent)
    oa = orc.get_state()["agent"].copy()
    oa[:, 5] = draw if envs is None else draw[envs]
    orc.set_state(agent=oa)


@pytest.mark.parametrize("R", [1, 2, 3])
def test_mini_benchmark(R, monkeypatch, capfd):
    """R desynchronised DoorKey-8x8 batches stepped in rotation through an action table of T rows, W eager warm-up steps,
    graphs of R * 5 steps and K not a multiple of G (the remainder graph runs too). Two CTAs per batch, so that the
    order list is in use; each graph holds 5 launches of every batch, so the frozen order direction does not alternate
    across replays."""
    env_id, n, T, W = "MiniGrid-DoorKey-8x8-v0", 2085, 7, 3
    G = 5 * R
    K = 2 * G + 2
    case = f"mini-bench/R={R}"
    envs, orcs = [], []
    for b in range(R):
        env, plan = make_engine(env_id, n, "next_step", monkeypatch, capfd, grid=2)
        check_plan(case, plan, env_id, n, TILED, grid=2)
        assert_order_list_live(case, plan, "next_step")
        orc = make_oracle(env_id, n, "next_step")
        env.reset(seed=1_000_003 * b)
        orc.reset(seed=1_000_003 * b)
        desync_both(env, orc, 77 + 1000 * b)
        envs.append(env)
        orcs.append(orc)
    acts, a_np = random_actions(T, n, seed=1234)
    rows_run = mini_bench(case, envs, [acts[i] for i in range(T)], T, W, G, K)
    for b in range(R):
        ends = 0
        for row in rows_run[b]:
            o = orcs[b].step(a_np[row])
            ends += int((o[3] | o[4]).sum())
        check_outputs(f"{case} batch {b}", f"last step ({len(rows_run[b])} steps)", engine_outputs(envs[b]), o)
        check_state(f"{case} batch {b}", "at the end", envs[b], orcs[b])
        assert ends > 0, f"{case} batch {b}: no episode ended"


def first_bad(case, where, what, ok):
    """ok: bool per env (or per env and element): names the first env, and its tile, for which it is False."""
    ok = np.asarray(ok).reshape(len(ok), -1).all(axis=1)
    if not ok.all():
        e = int(np.argmin(ok))
        raise AssertionError(f"{case}: {where}: {what} fails for {int((~ok).sum())} envs, the first env {e} (tile {e // 32})")


def check_whole_batch(case, where, env, out):
    """test_full_size_properties' invariants on every env of the batch."""
    obs, d, r, te, _ = out
    te = te.astype(bool)
    first_bad(case, where, "obs type <= 9, colour <= 5, state <= 2", (obs[..., 0] <= 9) & (obs[..., 1] <= 5) & (obs[..., 2] <= 2))
    first_bad(case, where, "reward in [0, 1], 0 unless terminated", (r >= 0) & (r <= 1) & (te | (r == 0)))
    first_bad(case, where, "direction in 0..3", (d >= 0) & (d <= 3))
    first_bad(case, where, "the agent's own cell is visible", obs[:, 3, 6, 0] != 0)
    st = engine_state(env)
    first_bad(case, where, "step_count <= max_steps", st["agent"][:, 5] <= env.max_steps)
    env.gen_obs()
    first_diff(case, f"{where}, gen_obs against the step's output", "obs", env._image.cpu().numpy(), obs)
    first_diff(case, f"{where}, gen_obs against the step's output", "dir", env._direction.cpu().numpy(), d)
    full = env.full_obs().cpu().numpy()
    cell = full[np.arange(env.num_envs), st["agent"][:, 0], st["agent"][:, 1]]
    first_bad(case, where, "full_obs holds (agent, red, dir) at the agent's cell", (cell[:, 0] == 10) & (cell[:, 2] == st["agent"][:, 2]))


def test_full_size_benchmark_graph(monkeypatch, capfd):
    """The headline shape: 2 x 262144 DoorKey-8x8 envs, 128-step graphs replayed twice (the warm replay and one
    timed one). A sample of 1024 envs (the first and last tiles and a stride) exactly against an oracle of those envs;
    the whole batch through invariants. Every CTA has more tiles than warps, so the order list is in use."""
    env_id, n, R, T, W, G = "MiniGrid-DoorKey-8x8-v0", 262144, 2, 64, 3, 128
    case = "full-size"
    sample = np.unique(np.concatenate([np.arange(32), np.arange(n - 32, n), np.arange(32, n - 32, 271)[:960]]))
    envs, orcs = [], []
    for b in range(R):
        env, plan = make_engine(env_id, n, "next_step", monkeypatch, capfd)
        check_plan(case, plan, env_id, n, TILED)
        assert_order_list_live(case, plan, "next_step")
        orc = OracleVecEnv(env_id, len(sample), autoreset="next_step", n_threads=0)
        env.reset(seed=1_000_003 * b)
        orc.reset(seed=(np.uint64(1_000_003 * b) + sample.astype(np.uint64)))
        desync_both(env, orc, 77 + 1000 * b, envs=sample)
        envs.append(env)
        orcs.append(orc)
    acts, a_np = random_actions(T, n, seed=1234)
    a_np = a_np[:, sample]
    rows_run = mini_bench(case, envs, [acts[i] for i in range(T)], T, W, G, G)
    for b in range(R):
        ends = 0
        for row in rows_run[b]:
            o = orcs[b].step(a_np[row])
            ends += int((o[3] | o[4]).sum())
        out = engine_outputs(envs[b])
        check_outputs(f"{case} batch {b}", f"last step ({len(rows_run[b])} steps)", [x[sample] for x in out], o, envs=sample)
        check_state(f"{case} batch {b}", "at the end", envs[b], orcs[b], envs=sample)
        assert ends > 0, f"{case} batch {b}: no episode ended in the sample"
        check_whole_batch(f"{case} batch {b}", f"last step ({len(rows_run[b])} steps)", envs[b], out)


# ---- 4. unaligned outputs outside the step ----
@pytest.mark.parametrize("env_id,layout", [("MiniGrid-DoorKey-8x8-v0", TILED), ("MiniGrid-FourRooms-v0", WINDOW)])
def test_unaligned_outputs_outside_the_step(env_id, layout, monkeypatch, capfd):
    """mg_gen_obs, mg_reset and mg_reset_masked write observations at every offset 1..15 (mod 16), enqueued back to back;
    a masked reset leaves the slots of the envs it does not reset untouched."""
    case = f"unaligned/{env_id}"
    n = 4133
    env, plan = make_engine(env_id, n, "next_step", monkeypatch, capfd)
    check_plan(case, plan, env_id, n, layout)
    orc = make_oracle(env_id, n, "next_step")
    env.reset(seed=900)
    orc.reset(seed=900)
    inject_ends(env, orc, n, 8, (), 1, seed=8)
    a = np.random.default_rng(9).integers(0, 7, n).astype(np.int32)
    env.step(torch.as_tensor(a, device="cuda"))  # a state that is not a fresh reset, with pending NEXT_STEP resets
    orc.step(a)
    ops = ["gen_obs", "reset", "reset_masked"] * 5
    obs, dirs = Guarded(15, n * 147, tuple(range(1, 16))), Guarded(15, n * 4, (4, 8, 12))
    rng = np.random.default_rng(10)
    masks = [rng.random(n) < 0.4 for _ in ops]
    masks_dev = [torch.as_tensor(m.astype(np.uint8), device="cuda") for m in masks]
    L, want = _lib.load(), []
    for i, op in enumerate(ops):
        if op == "gen_obs":
            _lib.check(L.mg_gen_obs(env._h, obs.ptr(i), dirs.ptr(i), stream()))
            want.append(copy_outputs(orc.gen_obs()))
        elif op == "reset":
            _lib.check(L.mg_reset(env._h, obs.ptr(i), dirs.ptr(i), stream()))
            want.append(copy_outputs(orc.reset()))
        else:
            _lib.check(L.mg_reset_masked(env._h, masks_dev[i].data_ptr(), obs.ptr(i), dirs.ptr(i), stream()))
            want.append(copy_outputs(orc.reset(mask=masks[i])))
    torch.cuda.synchronize()
    obs.fetch()
    dirs.fetch()
    for i, op in enumerate(ops):
        o = obs.slot(i, np.uint8).reshape(n, 7, 7, 3)
        d = dirs.slot(i, np.int32)
        sel = masks[i] if op == "reset_masked" else np.ones(n, bool)
        envs = np.nonzero(sel)[0]
        where = f"{op} into offset {obs.ptr(i) % 16}"
        first_diff(case, where, "obs", o[sel], want[i][0][sel], envs)
        first_diff(case, where, "dir", d[sel], want[i][1][sel].astype(np.int32), envs)
        assert (o[~sel] == CANARY).all() and (d[~sel].view(np.uint8) == CANARY).all(), \
            f"{case}: {where}: the slots of envs outside the mask were written"
    assert obs.residues() == set(range(1, 16))
    obs.check_canaries(f"{case}: obs")
    dirs.check_canaries(f"{case}: dir")
    check_state(case, "at the end", env, orc)


# ---- 5. more tiles per CTA than the order list holds ----
@pytest.mark.parametrize("env_id,layout,cfg", [("MiniGrid-DoorKey-8x8-v0", TILED, None), ("MiniGrid-DoorKey-8x8-v0", TILED, "0,0,2"),
                                               ("MiniGrid-FourRooms-v0", WINDOW, None)], ids=["tiled1", "tiled2", "window"])
def test_past_order_cap(env_id, layout, cfg, monkeypatch, capfd):
    """One CTA for 1251 tiles (NEXT_STEP: the order list exists only there). Tiles 0..1023 go through the list,
    flagged first; tiles 1024.. are pulled in index order behind it. Ends are forced on both sides of list index 1024."""
    n, T = 40013, 24
    case = f"order-cap/{env_id}/{cfg or 'default'}"
    env, plan = make_engine(env_id, n, "next_step", monkeypatch, capfd, cfg=cfg, grid=1)
    check_plan(case, plan, env_id, n, layout, cfg, 1)
    assert plan["grid"] == 1 and plan["tiles"] == 1251
    orc = make_oracle(env_id, n, "next_step")
    env.reset(seed=1100)
    orc.reset(seed=1100)
    wave_k = 9
    inject_ends(env, orc, n, T - 4, (3, 1000, 1023, 1024, 1100, 1249, 1250), wave_k, seed=11)
    acts, a_np = random_actions(T, n, seed=12)
    slots = Slots(T, n)
    want = run_chain_and_compare(case, env, orc, acts, a_np, T, slots)
    assert_resets_inside(case, want, n, wave_k - 1)
    per = np.stack([ends_per_tile(o, n) for o in want[:-1]])  # NEXT_STEP: an end before the last step resets in the chain
    assert per[:, :1024].sum() > 0 and per[:, 1024:].sum() > 0, f"{case}: resets must happen on both sides of the list cap"
    assert min(per[wave_k - 1, 1023], per[wave_k - 1, 1024]) >= DENSE_RESET_MIN, f"{case}: the waves at tiles 1023 / 1024"


# ---- 6. concurrent and interleaved handles ----
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
@pytest.mark.parametrize("streams", ["two-streams", "one-stream"])
def test_two_handles(streams, mode, monkeypatch, capfd):
    """DoorKey-8x8 and FourRooms chains enqueued alternately: on two streams (two K1 grids share the GPU) or on one
    (the benchmark's rotation of batches)."""
    n, T = 20000, 32
    case = f"two-handles/{streams}/{mode}"
    ids = (("MiniGrid-DoorKey-8x8-v0", TILED), ("MiniGrid-FourRooms-v0", WINDOW))
    envs, orcs, acts, slots = [], [], [], []
    for k, (env_id, layout) in enumerate(ids):
        env, plan = make_engine(env_id, n, mode, monkeypatch, capfd)
        check_plan(case, plan, env_id, n, layout)
        orc = make_oracle(env_id, n, mode)
        env.reset(seed=1200 + k)
        orc.reset(seed=1200 + k)
        inject_ends(env, orc, n, T - 4, (7, 400), 10, seed=13 + k)
        envs.append(env)
        orcs.append(orc)
        acts.append(random_actions(T, n, seed=14 + k))
        slots.append(Slots(T, n))
    cur = torch.cuda.current_stream()
    side = [torch.cuda.Stream(), torch.cuda.Stream()] if streams == "two-streams" else [cur, cur]
    for s in side:
        if s is not cur:
            s.wait_stream(cur)
    for t in range(T):
        for k in range(2):
            with torch.cuda.stream(side[k]):
                step_into(envs[k], acts[k][0][t], slots[k], t)
    for s in side:
        s.synchronize()
    torch.cuda.synchronize()
    for k in range(2):
        c = f"{case}: {ids[k][0]}"
        slots[k].fetch()
        want = []
        for t in range(T):
            o = copy_outputs(orcs[k].step(acts[k][1][t]))
            check_outputs(c, f"step {t}", slots[k].outputs(t), o)
            want.append(o)
        check_state(c, f"after {T} steps", envs[k], orcs[k])
        slots[k].check_canaries(c)
        slots[k].assert_mixed_alignment(c)
        assert_resets_inside(c, want, n, 9)


# ---- 7. consumers between steps ----
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
@pytest.mark.parametrize("env_id,layout", [("MiniGrid-DoorKey-8x8-v0", TILED), ("MiniGrid-FourRooms-v0", WINDOW)])
def test_consumers_between_steps(env_id, layout, mode, monkeypatch, capfd):
    """After every step of the chain, with no synchronisation: full_obs (K3), the 9 x 9 view (ViewSizeWrapper's kernel,
    through the C-ABI: the wrapper reuses one buffer) and the state hash (K4), each into its own slot."""
    n, T, V = 4133, 24, 9
    case = f"consumers/{env_id}/{mode}"
    env, plan = make_engine(env_id, n, mode, monkeypatch, capfd)
    check_plan(case, plan, env_id, n, layout)
    orc = hs.HashedOracle(env_id, n, autoreset=mode)
    env.reset(seed=1300)
    orc.reset(seed=1300)
    inject_ends(env, orc, n, T - 4, (2, 129), 7, seed=15)
    acts, a_np = random_actions(T, n, seed=16)
    W, H = env.width, env.height
    slots = Slots(T, n)
    full = Guarded(T, n * W * H * 3, OBS_RESIDUES)
    view = Guarded(T, n * V * V * 3, (3, 0, 7, 12, 1))
    digest = Guarded(T, n * 32, (0, 1, 5, 8, 15))
    L = _lib.load()
    for t in range(T):
        step_into(env, acts[t], slots, t)
        env.full_obs(out=full.tensor(t).view(n, W, H, 3))
        _lib.check(L.mg_obs_view(env._h, V, view.ptr(t), stream()))
        env.hash_digest(out=digest.tensor(t).view(n, 32))
    torch.cuda.synchronize()
    for g in (full, view, digest):
        g.fetch()
    slots.fetch()
    hashed = np.concatenate([np.arange(32), np.arange((n - 1) // 32 * 32, n)])  # the first and the (ragged) last tile
    want = []
    for t in range(T):
        o = copy_outputs(orc.step(a_np[t]))
        where = f"step {t}"
        check_outputs(case, where, slots.outputs(t), o)
        first_diff(case, where, "full_obs", full.slot(t, np.uint8).reshape(n, W, H, 3), orc.o.full_obs())
        first_diff(case, where, f"view {V}", view.slot(t, np.uint8).reshape(n, V, V, 3), orc.o.gen_obs_view(V))
        got = digest.slot(t, np.uint8).reshape(n, 32)
        want_hex = orc.hash(64, envs=hashed)
        for i, h in zip(hashed, want_hex):
            assert got[i].tobytes().hex() == h, f"{case}: {where}: hash of env {i} (tile {i // 32})"
        want.append(o)
    check_state(case, f"after {T} steps", env, orc)
    slots.check_canaries(case)
    for g, name in ((full, "full_obs"), (view, "view"), (digest, "hash")):
        g.check_canaries(f"{case}: {name} slots")
    slots.assert_mixed_alignment(case)
    assert_resets_inside(case, want, n, 6)
