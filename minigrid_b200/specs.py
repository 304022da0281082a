"""Registered ids -> constructor arguments of the four generators the engine implements.

Restated from the reference's registry and constructors (no code copied; citations relative to
/root/reference/minigrid/): __init__.py:25-28 (LavaCrossingS9N1), :106-109 (DoorKey-8x8), :159-162
(Empty-5x5), :183-185 (Empty-8x8), :214-216 (FourRooms); defaults empty.py:69-90 (max_steps 4*size^2,
see_through_walls=True), doorkey.py:62-68 (10*size^2), crossing.py:89-116 (4*size^2), fourrooms.py:55-67
(19x19, max_steps 100).
"""
from __future__ import annotations

from dataclasses import dataclass, field

KIND_EMPTY, KIND_DOORKEY, KIND_CROSSING, KIND_FOURROOMS, KIND_LAVAGAP, KIND_DISTSHIFT, KIND_MULTIROOM = 0, 1, 2, 3, 4, 5, 6
KIND_LOCKEDROOM, KIND_PLAYGROUND = 7, 8
KIND_GOTODOOR, KIND_FETCH, KIND_REDBLUEDOORS, KIND_GOTOOBJECT, KIND_PUTNEAR, KIND_MEMORY = 9, 10, 11, 12, 13, 14
KIND_DYNOBS = 15
KIND_ROOMGRID = 16
T_WALL, T_LAVA = 2, 9


@dataclass(frozen=True)
class EnvSpec:
    kind: int
    width: int
    height: int
    max_steps: int
    see_through_walls: bool
    params: tuple = field(default_factory=tuple)
    mission: str = ""


def empty(size=8, agent_start_pos=(1, 1), agent_start_dir=0, max_steps=None):
    random_start = agent_start_pos is None
    sx, sy = (0, 0) if random_start else agent_start_pos
    return EnvSpec(KIND_EMPTY, size, size, max_steps or 4 * size * size, True,
                   (int(random_start), sx, sy, agent_start_dir), "get to the green goal square")


def doorkey(size=8, max_steps=None):
    return EnvSpec(KIND_DOORKEY, size, size, max_steps or 10 * size * size, False, (),
                   "use the key to open the door and then get to the goal")


def crossing(size=9, num_crossings=1, obstacle_type="lava", max_steps=None):
    lava = obstacle_type == "lava"
    return EnvSpec(KIND_CROSSING, size, size, max_steps or 4 * size * size, False,
                   (num_crossings, T_LAVA if lava else T_WALL),
                   "avoid the lava and get to the green goal square" if lava
                   else "find the opening and get to the green goal square")


def fourrooms(max_steps=100):
    return EnvSpec(KIND_FOURROOMS, 19, 19, max_steps, False, (), "reach the goal")


def lavagap(size, obstacle_type="lava", max_steps=None):
    """envs/lavagap.py:68-91 (4*size^2 steps, see_through_walls=False)."""
    lava = obstacle_type == "lava"
    return EnvSpec(KIND_LAVAGAP, size, size, max_steps or 4 * size * size, False, (T_LAVA if lava else T_WALL,),
                   "avoid the lava and get to the green goal square" if lava
                   else "find the opening and get to the green goal square")


def distshift(width=9, height=7, strip2_row=2, agent_start_pos=(1, 1), agent_start_dir=0, max_steps=None):
    """envs/distshift.py:63-92 (4*width*height steps, see_through_walls=True, fixed agent start)."""
    return EnvSpec(KIND_DISTSHIFT, width, height, max_steps or 4 * width * height, True,
                   (strip2_row, agent_start_pos[0], agent_start_pos[1], agent_start_dir), "get to the green goal square")


def multiroom(minNumRooms, maxNumRooms, maxRoomSize=10, max_steps=None):
    """envs/multiroom.py:77-115 (25 x 25, max_steps = maxNumRooms * 20)."""
    return EnvSpec(KIND_MULTIROOM, 25, 25, max_steps or maxNumRooms * 20, False, (minNumRooms, maxNumRooms, maxRoomSize),
                   "traverse the rooms to get to the goal")


def lockedroom(size=19, max_steps=None):
    """envs/lockedroom.py:74-90 (max_steps = 10 * size). The mission names the drawn colours; it is not produced here."""
    return EnvSpec(KIND_LOCKEDROOM, size, size, max_steps or 10 * size, False, (),
                   "get the {lockedroom_color} key from the {keyroom_color} room, unlock the {door_color} door and go to the goal")


def playground(max_steps=100):
    """envs/playground.py:16-31 (19 x 19, max_steps 100, empty mission)."""
    return EnvSpec(KIND_PLAYGROUND, 19, 19, max_steps, False, (), "")


def gotodoor(size=5, max_steps=None):
    """envs/gotodoor.py:65-86. The mission names the target door's colour; it is not produced here."""
    return EnvSpec(KIND_GOTODOOR, size, size, max_steps or 4 * size * size, True, (), "go to the {color} door")


def fetch(size=8, numObjs=3, max_steps=None):
    """envs/fetch.py:72-103."""
    return EnvSpec(KIND_FETCH, size, size, max_steps or 5 * size * size, True, (numObjs,), "{syntax} {color} {type}")


def redbluedoors(size=8, max_steps=None):
    """envs/redbluedoors.py:60-72: the grid is 2 * size wide."""
    return EnvSpec(KIND_REDBLUEDOORS, 2 * size, size, max_steps or 20 * size * size, False, (),
                   "open the red door then the blue door")


def gotoobject(size=6, numObjs=2, max_steps=None):
    """envs/gotoobject.py:66-90."""
    return EnvSpec(KIND_GOTOOBJECT, size, size, max_steps or 5 * size * size, True, (numObjs,), "go to the {color} {type}")


def putnear(size=6, numObjs=2, max_steps=None):
    """envs/putnear.py:66-92 (max_steps = 5 * size)."""
    return EnvSpec(KIND_PUTNEAR, size, size, max_steps or 5 * size, True, (numObjs,),
                   "put the {move_color} {move_type} near the {target_color} {target_type}")


def memory(size=8, random_length=False, max_steps=None):
    """envs/memory.py:67-88."""
    return EnvSpec(KIND_MEMORY, size, size, max_steps or 5 * size * size, False, (int(random_length),),
                   "go to the matching object at the end of the hallway")


def dynobstacles(size=8, agent_start_pos=(1, 1), agent_start_dir=0, n_obstacles=4, max_steps=None):
    """envs/dynamicobstacles.py:72-105 (4 * size^2 steps, see_through_walls=True; too many obstacles are reduced)."""
    n_obst = int(n_obstacles) if n_obstacles <= size / 2 + 1 else int(size / 2)
    random_start = agent_start_pos is None
    sx, sy = (0, 0) if random_start else agent_start_pos
    return EnvSpec(KIND_DYNOBS, size, size, max_steps or 4 * size * size, True,
                   (n_obst, int(random_start), sx, sy, agent_start_dir), "get to the green goal square")


def roomgrid(variant, room_size, num_rows, num_cols, max_steps, mission, extra=()):
    """core/roomgrid.py:66-100: width = (room_size - 1) * num_cols + 1, height likewise; see_through_walls=False."""
    return EnvSpec(KIND_ROOMGRID, (room_size - 1) * num_cols + 1, (room_size - 1) * num_rows + 1, max_steps, False,
                   (variant, room_size, num_rows, num_cols) + tuple(extra), mission)


def obstructedmaze(variant, num_rows, num_cols, num_rooms_visited, key_in_box, blocked, agent_room=(0, 0), num_quarters=0):
    """envs/obstructedmaze.py:79-105 (room_size 6, max_steps = 4 * num_rooms_visited * room_size^2), obstructedmaze_v1.py."""
    return roomgrid(variant, 6, num_rows, num_cols, 4 * num_rooms_visited * 36, "pick up the blue ball",
                    (int(key_in_box), int(blocked), agent_room[0] | (agent_room[1] << 4), num_quarters))


def keycorridor(room_size=6, num_rows=3, max_steps=None):
    """envs/keycorridor.py:73-97 (obj_type "ball", 3 columns, 30 * room_size^2 steps)."""
    return roomgrid(3, room_size, num_rows, 3, max_steps or 30 * room_size ** 2, "pick up the {color} ball")


REGISTRY = {
    # BASELINE.json configs
    "MiniGrid-Empty-5x5-v0": empty(size=5),
    "MiniGrid-Empty-8x8-v0": empty(size=8),
    "MiniGrid-DoorKey-8x8-v0": doorkey(size=8),
    "MiniGrid-LavaCrossingS9N1-v0": crossing(9, 1, "lava"),
    "MiniGrid-FourRooms-v0": fourrooms(),
    # other registered ids of the same generators (__init__.py:31-74,94-116,159-192)
    "MiniGrid-Empty-Random-5x5-v0": empty(size=5, agent_start_pos=None),
    "MiniGrid-Empty-6x6-v0": empty(size=6),
    "MiniGrid-Empty-Random-6x6-v0": empty(size=6, agent_start_pos=None),
    "MiniGrid-Empty-16x16-v0": empty(size=16),
    "MiniGrid-DoorKey-5x5-v0": doorkey(size=5),
    "MiniGrid-DoorKey-6x6-v0": doorkey(size=6),
    "MiniGrid-DoorKey-16x16-v0": doorkey(size=16),
    "MiniGrid-LavaCrossingS9N2-v0": crossing(9, 2, "lava"),
    "MiniGrid-LavaCrossingS9N3-v0": crossing(9, 3, "lava"),
    "MiniGrid-LavaCrossingS11N5-v0": crossing(11, 5, "lava"),
    "MiniGrid-SimpleCrossingS9N1-v0": crossing(9, 1, "wall"),
    "MiniGrid-SimpleCrossingS9N2-v0": crossing(9, 2, "wall"),
    "MiniGrid-SimpleCrossingS9N3-v0": crossing(9, 3, "wall"),
    "MiniGrid-SimpleCrossingS11N5-v0": crossing(11, 5, "wall"),
    # round-1 widening (SURVEY 8f-1): base-step-only generators, __init__.py:79-88,295-310
    "MiniGrid-LavaGapS5-v0": lavagap(5),
    "MiniGrid-LavaGapS6-v0": lavagap(6),
    "MiniGrid-LavaGapS7-v0": lavagap(7),
    "MiniGrid-DistShift1-v0": distshift(strip2_row=2),
    "MiniGrid-DistShift2-v0": distshift(strip2_row=5),
    # __init__.py:363-385 (N4-S5-v0 is registered with 6 rooms: "legacy, misconfigured")
    "MiniGrid-MultiRoom-N2-S4-v0": multiroom(2, 2, 4),
    "MiniGrid-MultiRoom-N4-S5-v0": multiroom(6, 6, 5),
    "MiniGrid-MultiRoom-N4-S5-v1": multiroom(4, 4, 5),
    "MiniGrid-MultiRoom-N6-v0": multiroom(6, 6),
    # __init__.py:312-318, :516-522
    "MiniGrid-LockedRoom-v0": lockedroom(),
    "MiniGrid-Playground-v0": playground(),
    # generator + step post-filter: __init__.py:218-236, 241-250, 196-208, 527-537, 541-551, 323-357
    "MiniGrid-GoToDoor-5x5-v0": gotodoor(5),
    "MiniGrid-GoToDoor-6x6-v0": gotodoor(6),
    "MiniGrid-GoToDoor-8x8-v0": gotodoor(8),
    "MiniGrid-GoToObject-6x6-N2-v0": gotoobject(6, 2),
    "MiniGrid-GoToObject-8x8-N2-v0": gotoobject(8, 2),
    "MiniGrid-Fetch-5x5-N2-v0": fetch(5, 2),
    "MiniGrid-Fetch-6x6-N2-v0": fetch(6, 2),
    "MiniGrid-Fetch-8x8-N3-v0": fetch(8, 3),
    "MiniGrid-PutNear-6x6-N2-v0": putnear(6, 2),
    "MiniGrid-PutNear-8x8-N3-v0": putnear(8, 3),
    "MiniGrid-RedBlueDoors-6x6-v0": redbluedoors(6),
    "MiniGrid-RedBlueDoors-8x8-v0": redbluedoors(8),
    "MiniGrid-MemoryS17Random-v0": memory(17, True),
    "MiniGrid-MemoryS13Random-v0": memory(13, True),
    "MiniGrid-MemoryS13-v0": memory(13),
    "MiniGrid-MemoryS11-v0": memory(11),
    "MiniGrid-MemoryS9-v0": memory(9),
    "MiniGrid-MemoryS7-v0": memory(7),
    # RNG inside step: __init__.py:117-153
    "MiniGrid-Dynamic-Obstacles-5x5-v0": dynobstacles(5, n_obstacles=2),
    "MiniGrid-Dynamic-Obstacles-Random-5x5-v0": dynobstacles(5, agent_start_pos=None, n_obstacles=2),
    "MiniGrid-Dynamic-Obstacles-6x6-v0": dynobstacles(6, n_obstacles=3),
    "MiniGrid-Dynamic-Obstacles-Random-6x6-v0": dynobstacles(6, agent_start_pos=None, n_obstacles=3),
    "MiniGrid-Dynamic-Obstacles-8x8-v0": dynobstacles(8),
    "MiniGrid-Dynamic-Obstacles-16x16-v0": dynobstacles(16, n_obstacles=8),
    # RoomGrid family: __init__.py:12-20, 252-290, 555-563 (unlock.py:55-70: 8 * 36 steps; blockedunlockpickup.py:67-85: 16 * 36)
    "MiniGrid-Unlock-v0": roomgrid(0, 6, 1, 2, 288, "open the door"),
    "MiniGrid-UnlockPickup-v0": roomgrid(1, 6, 1, 2, 288, "pick up the {color} box"),
    "MiniGrid-BlockedUnlockPickup-v0": roomgrid(2, 6, 1, 2, 576, "pick up the {color} {type}"),
    "MiniGrid-KeyCorridorS3R1-v0": keycorridor(3, 1),
    "MiniGrid-KeyCorridorS3R2-v0": keycorridor(3, 2),
    "MiniGrid-KeyCorridorS3R3-v0": keycorridor(3, 3),
    "MiniGrid-KeyCorridorS4R3-v0": keycorridor(4, 3),
    "MiniGrid-KeyCorridorS5R3-v0": keycorridor(5, 3),
    "MiniGrid-KeyCorridorS6R3-v0": keycorridor(6, 3),
    # ObstructedMaze: __init__.py:387-514 (boxes hide keys: Box.contains)
    "MiniGrid-ObstructedMaze-1Dl-v0": obstructedmaze(4, 1, 2, 2, False, False),
    "MiniGrid-ObstructedMaze-1Dlh-v0": obstructedmaze(4, 1, 2, 2, True, False),
    "MiniGrid-ObstructedMaze-1Dlhb-v0": obstructedmaze(4, 1, 2, 2, True, True),
    "MiniGrid-ObstructedMaze-2Dl-v0": obstructedmaze(5, 3, 3, 4, False, False, (2, 1), 1),
    "MiniGrid-ObstructedMaze-2Dlh-v0": obstructedmaze(5, 3, 3, 4, True, False, (2, 1), 1),
    "MiniGrid-ObstructedMaze-2Dlhb-v0": obstructedmaze(5, 3, 3, 4, True, True, (2, 1), 1),
    "MiniGrid-ObstructedMaze-1Q-v0": obstructedmaze(5, 3, 3, 5, True, True, (1, 1), 1),
    "MiniGrid-ObstructedMaze-2Q-v0": obstructedmaze(5, 3, 3, 11, True, True, (2, 1), 2),
    "MiniGrid-ObstructedMaze-Full-v0": obstructedmaze(5, 3, 3, 25, True, True, (1, 1), 4),
    "MiniGrid-ObstructedMaze-2Dlhb-v1": obstructedmaze(6, 3, 3, 4, True, True, (2, 1), 1),
    "MiniGrid-ObstructedMaze-1Q-v1": obstructedmaze(6, 3, 3, 5, True, True, (1, 1), 1),
    "MiniGrid-ObstructedMaze-2Q-v1": obstructedmaze(6, 3, 3, 11, True, True, (2, 1), 2),
    "MiniGrid-ObstructedMaze-Full-v1": obstructedmaze(6, 3, 3, 25, True, True, (1, 1), 4),
}


BABYAI_GOTO = 7  # roomgrid variant of the one-room BabyAI GoTo levels
BABYAI_REDBALL_GREY, BABYAI_REDBALL, BABYAI_OBJ, BABYAI_LOCAL, BABYAI_REDBLUEBALL = 0, 1, 2, 3, 4


def babyai_goto(level, room_size=8, num_dists=7, mission="go to {article} {color} {type}"):
    """envs/babyai/goto.py on one room (babyai/core/roomgrid_level.py:46-85): max_steps = room_size^2 (one navigation).
    The mission names the drawn target, and says "a" instead of "the" when several objects match it; a constant string
    only where the level makes it one."""
    return roomgrid(BABYAI_GOTO, room_size, 1, 1, room_size * room_size, mission, (level, num_dists))


# __init__.py:573-665 (the BabyAI GoTo levels that fit in one room)
BABYAI_REGISTRY = {
    "BabyAI-GoToRedBallGrey-v0": babyai_goto(BABYAI_REDBALL_GREY, mission="go to the red ball"),
    "BabyAI-GoToRedBall-v0": babyai_goto(BABYAI_REDBALL, mission="go to {article} red ball"),
    "BabyAI-GoToRedBallNoDists-v0": babyai_goto(BABYAI_REDBALL, num_dists=0, mission="go to the red ball"),
    "BabyAI-GoToObj-v0": babyai_goto(BABYAI_OBJ, num_dists=1, mission="go to the {color} {type}"),
    "BabyAI-GoToObjS4-v0": babyai_goto(BABYAI_OBJ, 4, 1, "go to the {color} {type}"),
    "BabyAI-GoToObjS6-v1": babyai_goto(BABYAI_OBJ, 6, 1, "go to the {color} {type}"),
    "BabyAI-GoToLocal-v0": babyai_goto(BABYAI_LOCAL, num_dists=8),
    **{f"BabyAI-GoToLocalS{s}N{n}-v0": babyai_goto(BABYAI_LOCAL, s, n)
       for s, n in [(5, 2), (6, 2), (6, 3), (6, 4), (7, 4), (7, 5), (8, 2), (8, 3), (8, 4), (8, 5), (8, 6), (8, 7)]},
    # the distractors are never red or blue balls, so the target is the only match
    "BabyAI-GoToRedBlueBall-v0": babyai_goto(BABYAI_REDBLUEBALL, mission="go to the {color} ball"),
}


BABYAI_PICKUP_PUTNEXT = 8  # roomgrid variant of the one-room BabyAI Pickup and PutNext levels
BABYAI_ONEROOM, BABYAI_PICKUPDIST, BABYAI_PUTNEXTLOCAL = 0, 1, 2


def babyai_pickup_putnext(level, room_size, num_objs, num_navs, mission, strict=False):
    """envs/babyai/other.py (OneRoomS*), pickup.py (PickupDist), putnext.py (PutNextLocal) on one room: max_steps =
    num_navs * room_size^2 (roomgrid_level.py:71-85; PutNextInstr needs two navigations). PickupDist's mission drops the
    colour or says "object" instead of the type, as its drawn descriptor does."""
    return roomgrid(BABYAI_PICKUP_PUTNEXT, room_size, 1, 1, num_navs * room_size * room_size, mission,
                    (level, num_objs, int(strict)))


# __init__.py:864-873, 883-898, 1059-1081 (the BabyAI Pickup and PutNext levels that fit in one room)
BABYAI_PICKUP_PUTNEXT_REGISTRY = {
    **{f"BabyAI-OneRoomS{s}-v0": babyai_pickup_putnext(BABYAI_ONEROOM, s, 1, 1, "pick up the ball")
       for s in (8, 12, 16, 20)},
    "BabyAI-PickupDist-v0": babyai_pickup_putnext(BABYAI_PICKUPDIST, 7, 5, 1, "pick up {article} {color} {type}"),
    "BabyAI-PickupDistDebug-v0": babyai_pickup_putnext(BABYAI_PICKUPDIST, 7, 5, 1, "pick up {article} {color} {type}",
                                                       strict=True),
    "BabyAI-PutNextLocal-v0": babyai_pickup_putnext(BABYAI_PUTNEXTLOCAL, 8, 8, 2,
                                                    "put the {color} {type} next to the {color} {type}"),
    **{f"BabyAI-PutNextLocalS{s}N{n}-v0": babyai_pickup_putnext(BABYAI_PUTNEXTLOCAL, s, n, 2,
                                                                "put the {color} {type} next to the {color} {type}")
       for s, n in [(5, 3), (6, 4)]},
}


def get(env_id: str) -> EnvSpec:
    if env_id in BABYAI_REGISTRY:
        return BABYAI_REGISTRY[env_id]
    if env_id in BABYAI_PICKUP_PUTNEXT_REGISTRY:
        return BABYAI_PICKUP_PUTNEXT_REGISTRY[env_id]
    try:
        return REGISTRY[env_id]
    except KeyError:
        raise KeyError(f"{env_id!r} is not one of the ids this engine implements: "
                       f"{sorted(REGISTRY) + sorted(BABYAI_REGISTRY) + sorted(BABYAI_PICKUP_PUTNEXT_REGISTRY)}") from None
