"""Blueprint files: a fixed full-tree strategy saved for later play (`solve_game --save`, `exploitability --save`) and loaded by
`head_to_head --blueprint_a / --blueprint_b`, `local_br --blueprint` and `play --blueprint`.

One `.npz` holds
    num_dice, num_faces   the game
    strategy              the compact table [N - 1, H] fp64 (entry [child - 1, hand] over the full tree's BFS order, N = 2^A - 1)
    source                "solve_game", "to_leaf" or "every_node"
    settings              JSON of the settings that made it (solver, iterations, depth, net)
    br, exploitability    the table's best-response pair and (br0 + br1) / 2
"""
import json

import numpy as np

SOURCES = ("solve_game", "to_leaf", "every_node")
MAX_ACTIONS = 23   # CFRB_TO_LEAF_MAX_ACTIONS: no blueprint above it


def table_shape(num_dice, num_faces):
    """[N - 1, H] of a game's blueprint; games above 23 actions have none (ValueError)."""
    A = 1 + 2 * num_dice * num_faces
    if A > MAX_ACTIONS:
        raise ValueError(f"{num_dice}x{num_faces}f has {A} actions: games with more than {MAX_ACTIONS} actions have no blueprint")
    return (1 << A) - 2, num_faces ** num_dice


def save_blueprint(path, num_dice, num_faces, strategy, source, settings, br):
    """Write the file (exactly at `path`) and return the path."""
    if source not in SOURCES:
        raise ValueError(f"source must be one of {SOURCES}, not {source!r}")
    s = np.ascontiguousarray(np.asarray(strategy, dtype=np.float64))
    if s.shape != table_shape(num_dice, num_faces):
        raise ValueError(f"a {num_dice}x{num_faces}f blueprint is {list(table_shape(num_dice, num_faces))}, got {list(s.shape)}")
    br = [float(x) for x in br]
    with open(path, "wb") as f:
        np.savez(f, num_dice=np.int64(num_dice), num_faces=np.int64(num_faces), strategy=s, source=np.str_(source),
                 settings=np.str_(json.dumps(settings, sort_keys=True)), br=np.array(br), exploitability=np.float64((br[0] + br[1]) / 2))
    return path


def load_blueprint(path, num_dice, num_faces):
    """The file's contents as a dict; a file of another game or with a table of the wrong shape is refused (ValueError)."""
    shape = table_shape(num_dice, num_faces)
    with np.load(path, allow_pickle=False) as z:
        d, f = int(z["num_dice"]), int(z["num_faces"])
        if (d, f) != (num_dice, num_faces):
            raise ValueError(f"{path} holds a {d}x{f}f blueprint, not {num_dice}x{num_faces}f")
        s = np.ascontiguousarray(z["strategy"], dtype=np.float64)
        if s.shape != shape:
            raise ValueError(f"{path}: a {num_dice}x{num_faces}f blueprint is {list(shape)}, the file holds {list(s.shape)}")
        return {"num_dice": d, "num_faces": f, "strategy": s, "source": str(z["source"]), "settings": json.loads(str(z["settings"])),
                "br": [float(x) for x in z["br"]], "exploitability": float(z["exploitability"])}


def blueprint_name(path):
    """How report lines name a blueprint agent."""
    return "blueprint:" + path
