"""Seeded edit scripts over one layer, and what they imply for the engine (plain Python, no GPU).

A layer goes through many versions: `script(seed, n, bb)` is the list of operations that turns version k-1 into version
k, `apply` performs them, `freeze` keeps an exact copy of a version.  `expected_written` is DESIGN.md §6's diff rule
restated over the ORACLE's block tables: which blocks a diff pass must write.  `expected_pruned` is what VMIG_F_PRUNE
must remove.  `make_kind` builds one entry of each kind a path can have, for the kind-change matrix."""
import json
import os
import shutil
import stat
import subprocess
from pathlib import Path

import numpy as np

# ------------------------------------------------------------------------------------------------ names and kinds
# names tar, the walk and the block table must carry unharmed (str with surrogateescape: what os.fsdecode gives)
NAME_POOL = ["sp ace", "new\nline", "bad\udcff\udcfebyte", ".dot", "-dash", "tab\there", "q'uo\"te", "ümläut", "L" * 255]

KINDS = ("file", "empty", "emptydir", "dir", "symlink", "fifo", "hardlink")
SYMLINK_VARIANTS = ("file", "dir", "dangling")
# GNU tar replaces whatever is in the way of an entry, an empty directory included; only a non-empty directory stops it
TAR_REFUSES = {("dir", new) for new in KINDS if new not in ("dir", "emptydir")}
KIND_PAIRS_OK = [(a, b) for a in KINDS for b in KINDS if (a, b) not in TAR_REFUSES]


def awkward(i: int, tag: str = "", room: int = 0) -> str:
    """The i-th awkward name, made unique by its index; at most 255 - room bytes."""
    base = NAME_POOL[i % len(NAME_POOL)]
    tail = f"{tag}{i}"
    return os.fsdecode(os.fsencode(base)[:255 - room - len(tail)]) + tail


def data(seed: int, n: int) -> bytes:
    return np.random.default_rng(seed).bytes(n) if n else b""


def remove_any(p) -> None:
    p = os.fspath(p)
    if os.path.isdir(p) and not os.path.islink(p):
        shutil.rmtree(p)
    elif os.path.lexists(p):
        os.unlink(p)


def partner(path: str) -> str:
    """The second path of the hard-link pair a 'hardlink' kind makes (sorts after path: path is the group's primary)."""
    return path + ".p"


def make_kind(root, rel: str, kind: str, seed: int, size: int = 5000) -> None:
    """Put an entry of `kind` at root/rel, replacing whatever is there.  seed picks the content, the directory's
    children and the symlink variant, so that two calls with different seeds differ in what a copy must carry."""
    p = os.path.join(os.fspath(root), rel)
    remove_any(p)
    if kind == "file":
        Path(p).write_bytes(data(seed, size + seed % 7))
    elif kind == "empty":
        Path(p).write_bytes(b"")
    elif kind == "emptydir":
        os.mkdir(p)
    elif kind == "dir":
        os.mkdir(p)
        Path(p, f"c{seed % 3}").write_bytes(data(seed + 1, 300))
        os.mkdir(os.path.join(p, "sub"))
        os.symlink("../gone", os.path.join(p, "sub", "l"))
    elif kind == "symlink":
        v = SYMLINK_VARIANTS[seed % 3]
        os.symlink({"file": "../f/target", "dir": "..", "dangling": f"/nonexistent/{seed}"}[v], p)
    elif kind == "fifo":
        os.mkfifo(p, 0o640 if seed % 2 else 0o600)
    elif kind == "hardlink":
        Path(p).write_bytes(data(seed, size + seed % 5))
        remove_any(partner(p))
        os.link(p, partner(p))
    else:
        raise ValueError(kind)


def kind_at(p) -> str:
    """The kind, in KINDS' terms, of what sits at p."""
    st = os.lstat(p)
    if stat.S_ISDIR(st.st_mode):
        return "dir" if os.listdir(p) else "emptydir"
    if stat.S_ISREG(st.st_mode):
        return "hardlink" if st.st_nlink > 1 else "file" if st.st_size else "empty"
    return {stat.S_IFLNK: "symlink", stat.S_IFIFO: "fifo"}[stat.S_IFMT(st.st_mode)]


KIND_PATH = "k/x"


def kind_tree(root, kind: str, seed: int) -> None:
    """A small tree whose KIND_PATH is of `kind`, next to a file every such tree has."""
    root = Path(root)
    (root / "f").mkdir(parents=True)
    (root / "k").mkdir()
    (root / "f" / "target").write_bytes(b"symlinks point here")
    (root / "k" / "keep").write_bytes(data(5, 70000))
    os.utime(root / "k" / "keep", ns=(10**18, 10**18))
    make_kind(root, KIND_PATH, kind, seed)


# ------------------------------------------------------------------------------------------------ the initial layer
def layer_sizes(bb: int):
    return [0, 1, bb - 1, bb, bb + 1, 3 * bb + 5, 9 * bb]


def kind_slots():
    """One path under k/ for every kind pair tar carries out: slot i starts as pair[0] and becomes pair[1] once."""
    return [(f"k/{awkward(i, 'k', room=2)}", a, b) for i, (a, b) in enumerate(KIND_PAIRS_OK)]


def build_layer(root, orc, bb: int, make_rich_tree) -> None:
    root = Path(root)
    (root / "rich").mkdir(parents=True)
    make_rich_tree(root / "rich", orc)
    for d in ("f", "k", "d/n1/n2/n3", "d/empty"):
        (root / d).mkdir(parents=True)
    for i, size in enumerate(layer_sizes(bb)):
        (root / "f" / awkward(i, "s")).write_bytes(data(100 + i, size))
    (root / "f" / "target").write_bytes(b"symlinks point here")
    for n in ("dupA", "dupB"):
        (root / "f" / n).write_bytes(data(7, 2 * bb + 7))
    (root / "f" / "zeros").write_bytes(bytes(2 * bb))
    (root / READONLY).write_bytes(data(15, 2 * bb + 3))
    with open(root / "f" / "hole", "wb") as f:
        f.write(data(8, bb))
        f.seek(2 * bb)
        f.write(data(9, bb))
    (root / "f" / "t1").write_bytes(data(10, bb + 9))
    os.link(root / "f" / "t1", root / "f" / "t2")
    os.link(root / "f" / "t1", root / "d" / "t3")
    (root / "d" / "doomed" / "in" / "ner").mkdir(parents=True)
    (root / "d" / "doomed" / "in" / "a").write_bytes(data(14, 4097))
    os.symlink("a", root / "d" / "doomed" / "in" / "l")
    (root / "d" / "n1" / "x").write_bytes(data(11, bb + 100))
    (root / "d" / "n1" / "n2" / "y").write_bytes(data(12, 2 * bb))
    (root / "d" / "n1" / "n2" / "n3" / awkward(8, "z")).write_bytes(data(13, 777))
    for i, (rel, a, _b) in enumerate(kind_slots()):
        make_kind(root, rel, a, 1000 + i)


class _Model:
    """What the generator must know of the layer to pick operations that are valid: the single-link regular files it may
    edit (path -> size), the hard-link groups, the directory it renames and the kind every k/ slot has."""

    def __init__(self, bb: int):
        self.bb = bb
        self.files = {f"f/{awkward(i, 's')}": s for i, s in enumerate(layer_sizes(bb))}
        self.files.update({"f/dupA": 2 * bb + 7, "f/dupB": 2 * bb + 7, "f/zeros": 2 * bb, "f/hole": 3 * bb,
                           "d/n1/x": bb + 100, "d/n1/n2/y": 2 * bb})
        self.equal = [["f/dupA", "f/dupB"]]           # sets of single-link files known to hold the same bytes
        self.groups = [["f/t1", "f/t2", "d/t3"]]
        self.gsize = {0: bb + 9}
        self.ndir = "d/n1"                            # the directory rename_dir moves
        self.slots = {rel: a for rel, a, _ in kind_slots()}
        self.was_dir = {rel for rel, a, _ in kind_slots() if a == "dir"}
        self.fresh = 0

    def new_path(self) -> str:
        self.fresh += 1
        return f"f/{awkward(self.fresh, 'n')}"

    def forget_equal(self, path):
        self.equal = [[p for p in g if p != path] for g in self.equal]
        self.equal = [g for g in self.equal if len(g) > 1]

    def move(self, a, b):
        if a in self.files:
            self.files[b] = self.files.pop(a)
        self.equal = [[b if p == a else p for p in g] for g in self.equal]
        self.groups = [[b if p == a else p for p in g] for g in self.groups]


OP_CYCLE = [
    # content
    ("flip", "first"), ("flip", "last"), ("flip", "run"), ("poke_tail", ""), ("append", "within"), ("append", "across"),
    ("truncate", "multiple"), ("truncate", "mid"), ("truncate", "zero"), ("grow", ""), ("rewrite_same", ""),
    # identity without content
    ("replace_inode", "keep_mtime"), ("replace_inode", "new_mtime"), ("chmod", ""), ("chown", ""), ("utime", ""),
    # placement
    ("rename", ""), ("rename_dir", ""), ("swap", ""), ("cp", ""), ("rm", ""), ("rmtree", ""), ("cut_head", ""),
    # hard links
    ("link_add", ""), ("unlink_one", ""), ("break_link", ""), ("join", ""),
]
# What every seed applies whatever the shuffle says.  In-place truncation is the rule most likely to break.  READONLY
# exposed a divergence once: an ordinary user's engine could not patch, nor even leave alone, a destination file whose
# mode has no write bit, where tar replaces it.  It loses its write bit in the first version, changes one block in the
# second and stays as it is from then on.
FIXED_FIRST = [("truncate", "mid")]
READONLY = "f/readonly"


def _gen(m: _Model, rng, name: str, var: str) -> dict:
    bb = m.bb
    pick = lambda keys: sorted(keys)[int(rng.integers(len(keys)))]
    nonempty = [p for p, s in m.files.items() if s > 0]
    big = [p for p, s in m.files.items() if s > bb]
    seed = int(rng.integers(1 << 30))
    if name == "flip":
        p = pick(big)
        nb = -(-m.files[p] // bb)
        blocks = {"first": [0], "last": [nb - 1], "run": list(range(max(0, nb - 3), nb))}[var]
        m.forget_equal(p)
        return {"op": "flip", "var": var, "path": p, "blocks": blocks, "bb": bb}
    if name == "poke_tail":
        p = pick([q for q in nonempty if m.files[q] % bb])
        m.forget_equal(p)
        return {"op": "poke_tail", "path": p}
    if name == "append":
        p = pick([q for q in nonempty if (-m.files[q]) % bb > 1] if var == "within" else nonempty)
        room = (-m.files[p]) % bb
        n = room // 2 if var == "within" else room + bb // 2 + 3
        m.files[p] += n
        m.forget_equal(p)
        return {"op": "append", "var": var, "path": p, "n": n, "seed": seed}
    if name == "truncate":
        p = pick(big) if var != "zero" else pick(nonempty)
        whole = (m.files[p] - 1) // bb * bb           # the file without its last block, short or not
        size = {"multiple": whole, "mid": whole - bb // 3, "zero": 0}[var]
        m.files[p] = size
        m.forget_equal(p)
        return {"op": "truncate", "var": var, "path": p, "size": size}
    if name == "grow":
        empties = [p for p, s in m.files.items() if s == 0]
        p = pick(empties) if empties else m.new_path()
        m.files[p] = bb + 11
        return {"op": "grow", "path": p, "n": bb + 11, "seed": seed}
    if name == "rewrite_same":
        return {"op": "rewrite_same", "path": pick(nonempty)}
    if name == "replace_inode":
        return {"op": "replace_inode", "var": var, "path": pick(nonempty)}
    if name == "chmod":
        return {"op": "chmod", "path": pick(m.files), "mode": [0o600, 0o755, 0o4711, 0o444][seed % 4]}
    if name == "chown":
        return {"op": "chown", "path": pick(m.files), "uid": 1000 + seed % 5, "gid": 2000 + seed % 3}
    if name == "utime":
        return {"op": "utime", "path": pick(m.files), "ns": 1_600_000_000_000_000_000 + seed * 1_000_003}
    if name == "rename":
        a, b = pick(m.files), m.new_path()
        m.move(a, b)
        return {"op": "rename", "path": a, "to": b}
    if name == "rename_dir":
        a = m.ndir
        m.fresh += 1
        b = f"d/{awkward(m.fresh, 'r')}"
        for p in [p for g in [m.files] + m.groups + m.equal for p in g if p.startswith(a + "/")]:
            m.move(p, b + p[len(a):])
        m.ndir = b
        return {"op": "rename_dir", "path": a, "to": b}
    if name == "swap":
        a = pick(m.files)
        b = pick([p for p in m.files if p != a])
        m.files[a], m.files[b] = m.files[b], m.files[a]
        m.equal = [[{a: b, b: a}.get(p, p) for p in g] for g in m.equal]
        return {"op": "swap", "path": a, "with": b}
    if name == "cp":
        a, b = pick([p for p, s in m.files.items() if 0 < s <= 3 * bb + 5]), m.new_path()
        m.files[b] = m.files[a]
        for g in m.equal:
            if a in g:
                g.append(b)
                break
        else:
            m.equal.append([a, b])
        return {"op": "cp", "path": a, "to": b}
    if name == "rm":
        p = pick(m.files)
        del m.files[p]
        m.forget_equal(p)
        return {"op": "rm", "path": p}
    if name == "rmtree":
        return {"op": "rmtree", "path": "d/doomed"}
    if name == "cut_head":
        p = pick(big)
        m.files[p] -= bb
        m.forget_equal(p)
        return {"op": "cut_head", "path": p, "n": bb}
    if name == "link_add":
        live = [i for i, g in enumerate(m.groups) if g]
        gi = live[int(rng.integers(len(live)))] if live and seed % 3 else -1
        b = m.new_path()
        if gi < 0:
            a = pick(nonempty)
            m.groups.append([a, b])
            m.gsize[len(m.groups) - 1] = m.files.pop(a)
            m.forget_equal(a)
        else:
            a = m.groups[gi][0]
            m.groups[gi].append(b)
        return {"op": "link_add", "path": a, "to": b}
    if name in ("unlink_one", "break_link"):
        pre = [] if any(m.groups) else [_gen(m, rng, "link_add", "")]      # no group left: make one first
        gi = [i for i, g in enumerate(m.groups) if g][0]
        g = m.groups[gi]
        p = g.pop(int(rng.integers(len(g))))
        if name == "break_link":
            m.files[p] = m.gsize[gi]
        if len(g) == 1:                               # the last path left is a plain file again
            m.files[g[0]] = m.gsize[gi]
            g.clear()
        return {"op": name, "path": p, "pre": pre}
    if name == "join":
        if not m.equal:
            a, b = pick([p for p, s in m.files.items() if 0 < s <= 3 * bb + 5]), m.new_path()
            m.files[b] = m.files[a]
            m.equal.append([a, b])
            pre = [{"op": "cp", "path": a, "to": b}]
        else:
            pre = []
        g = m.equal.pop(0)
        a, b = g[0], g[1]
        m.groups.append([a, b])
        m.gsize[len(m.groups) - 1] = m.files.pop(a)
        m.files.pop(b)
        for p in g[2:]:
            m.forget_equal(p)
        return {"op": "join", "path": a, "with": b, "pre": pre}
    raise ValueError(name)


def script(seed: int, n_versions: int = 8, bb: int = 65536) -> list:
    """One list of operations per version, deterministic in (seed, n_versions, bb) and JSON-able.  Every operation of
    OP_CYCLE appears at least once, and every kind pair of KIND_PAIRS_OK happens at its own k/ slot between two
    consecutive versions, so that each seed observes all of them."""
    rng = np.random.default_rng(seed)
    m = _Model(bb)
    slots = kind_slots()
    when = rng.permutation(len(slots)) % n_versions            # the version at which slot i makes its transition
    cycle = [OP_CYCLE[i] for i in rng.permutation(len(OP_CYCLE))]
    per = -(-len(cycle) // n_versions)
    out = []
    for v in range(n_versions):
        ops = []
        todo = (FIXED_FIRST if v == 0 else []) + cycle[v * per:(v + 1) * per]
        if v * per >= len(cycle):                              # more versions than the cycle fills: draw again
            todo = [OP_CYCLE[int(rng.integers(len(OP_CYCLE)))] for _ in range(per)]
        for name, var in todo:
            ops.append(_gen(m, rng, name, var))
        if v == 0:
            ops.append({"op": "chmod", "path": READONLY, "mode": 0o444})
        elif v == 1:
            ops.append({"op": "flip", "var": "readonly", "path": READONLY, "blocks": [1], "bb": bb})
        for i, (rel, a, b) in enumerate(slots):
            if when[i] == v:
                ops.append({"op": "set_kind", "path": rel, "was": a, "kind": b, "seed": int(rng.integers(1 << 20))})
                m.slots[rel] = b
                if b == "dir":
                    m.was_dir.add(rel)
        # a second change at a slot that already made its own: chains of kinds at one path.  A slot that ever was a
        # non-empty directory stays a directory: without VMIG_F_PRUNE the destination keeps the old children, and tar
        # refuses to put anything else there
        done = sorted(rel for i, (rel, _a, _b) in enumerate(slots) if when[i] < v and rel not in m.was_dir)
        if done:
            rel = done[int(rng.integers(len(done)))]
            b = [k for k in KINDS if k != "dir"][int(rng.integers(len(KINDS) - 1))]
            ops.append({"op": "set_kind", "path": rel, "was": m.slots[rel], "kind": b, "seed": int(rng.integers(1 << 20))})
            m.slots[rel] = b
        out.append(ops)
    json.dumps(out)
    return out


# ------------------------------------------------------------------------------------------------ apply and freeze
CONTENT_OPS = ("flip", "poke_tail", "append", "truncate", "grow", "rewrite_same", "cut_head")


def _rewrite(p, body: bytes):
    with open(p, "r+b") as f:
        f.write(body)


def apply(root, ops) -> None:
    root = os.fspath(root)
    P = lambda rel: os.path.join(root, rel)
    for o in ops:
        apply(root, o.get("pre", []))
        op, p = o["op"], P(o["path"])
        # an ordinary user edits a file of theirs that has no write bit by lending it one: the mode is part of the version
        mode = None
        if op in CONTENT_OPS and os.path.isfile(p) and not os.stat(p).st_mode & 0o200:
            mode = stat.S_IMODE(os.stat(p).st_mode)
            os.chmod(p, mode | 0o200)
        if op == "flip":
            with open(p, "r+b") as f:
                for b in o["blocks"]:
                    f.seek(b * o["bb"])
                    c = f.read(1)
                    f.seek(b * o["bb"])
                    f.write(bytes([c[0] ^ 0x5A]))
        elif op == "poke_tail":
            with open(p, "r+b") as f:
                f.seek(-1, os.SEEK_END)
                c = f.read(1)
                f.seek(-1, os.SEEK_END)
                f.write(bytes([c[0] ^ 0xA5]))
        elif op == "append":
            with open(p, "ab") as f:
                f.write(data(o["seed"], o["n"]))
        elif op == "truncate":
            os.truncate(p, o["size"])
        elif op == "grow":
            Path(p).write_bytes(data(o["seed"], o["n"]))
        elif op == "rewrite_same":
            _rewrite(p, Path(p).read_bytes())
        elif op == "replace_inode":
            st = os.lstat(p)
            shutil.copyfile(p, p + ".tmp")
            shutil.copystat(p, p + ".tmp")
            if os.geteuid() == 0:
                os.chown(p + ".tmp", st.st_uid, st.st_gid)
            if o["var"] == "new_mtime":
                os.utime(p + ".tmp", ns=(st.st_atime_ns, st.st_mtime_ns + 3_000_000_000))
            os.rename(p + ".tmp", p)
        elif op == "chmod":
            os.chmod(p, o["mode"])
        elif op == "chown":
            if os.geteuid() == 0:
                os.chown(p, o["uid"], o["gid"])
        elif op == "utime":
            os.utime(p, ns=(o["ns"], o["ns"]))
        elif op in ("rename", "rename_dir"):
            remove_any(P(o["to"]))
            os.rename(p, P(o["to"]))
        elif op == "swap":
            q = P(o["with"])
            os.rename(p, p + ".swap")
            os.rename(q, p)
            os.rename(p + ".swap", q)
        elif op == "cp":
            shutil.copyfile(p, P(o["to"]))
        elif op == "rm":
            os.unlink(p)
        elif op == "rmtree":
            remove_any(p)
        elif op == "cut_head":
            body = Path(p).read_bytes()[o["n"]:]
            Path(p).write_bytes(body)
        elif op == "link_add":
            os.link(p, P(o["to"]))
        elif op == "unlink_one":
            os.unlink(p)
        elif op == "break_link":
            body = Path(p).read_bytes()
            os.unlink(p)
            Path(p).write_bytes(body)
        elif op == "join":
            os.unlink(P(o["with"]))
            os.link(p, P(o["with"]))
        elif op == "set_kind":
            make_kind(root, o["path"], o["kind"], o["seed"])
        else:
            raise ValueError(op)
        if mode is not None:
            os.chmod(p, mode)


def freeze(root, dst) -> None:
    """An exact copy of root as the new directory dst: cp -a keeps hard links, owners, modes and nanosecond mtimes."""
    os.mkdir(dst)
    subprocess.run(["cp", "-a", os.path.join(os.fspath(root), "."), os.fspath(dst)], check=True)


# ------------------------------------------------------------------------------------------------ what a call must do
def tree_in_itself(orc, root, mtime_ns: bool = False) -> dict:
    """The oracle's manifest of root with hard-link groups as seen INSIDE the tree: a snapshot's file whose other links
    all live in other snapshots is a plain file here."""
    man = orc.tree_manifest(root, mtime_ns=mtime_ns)
    size = {}
    for r in man.values():
        if "hardlink_to" in r:
            size[r["hardlink_to"]] = size.get(r["hardlink_to"], 0) + 1
    for r in man.values():
        if "hardlink_to" in r and size[r["hardlink_to"]] < 2:
            del r["hardlink_to"]
    return man


def diff_manifests(a: dict, b: dict) -> list:
    return [(k, a.get(k), b.get(k)) for k in sorted(set(a) | set(b)) if a.get(k) != b.get(k)]


def secondaries(man: dict) -> set:
    """Paths (bytes, as block tables carry them) that are a later path of a hard-link group: never written, linked."""
    return {os.fsencode(rel) for rel, r in man.items() if r.get("hardlink_to", rel) != rel}


def single_files(man: dict) -> set:
    return {os.fsencode(rel) for rel, r in man.items() if stat.S_ISREG(r["type"]) and "hardlink_to" not in r}


def _blocks(table, bb):
    entries, hashes = table
    return {rel: [(int(hashes[first + i]), min(bb, size - i * bb)) for i in range(-(-size // bb))]
            for rel, size, first in entries}


def expected_written(table_prev, table_now, second_now: set, trusted: set, bb: int):
    """(blocks, bytes) a diff pass must write to turn what the destination holds into the source, by DESIGN.md §6: a
    file in `trusted` (a single-link regular file the previous call left at this path, recorded in table_prev) is
    patched in place and takes the blocks whose hash or length differs or that are new; every other file is written
    whole, a hard-link group once (second_now: the group's later paths).  Tables are the oracle's (entries, hashes)."""
    prev = _blocks(table_prev, bb) if table_prev else {}
    n = nbytes = 0
    for rel, blocks in _blocks(table_now, bb).items():
        if rel in second_now:
            continue
        old = prev.get(rel, []) if rel in trusted else []
        for i, blk in enumerate(blocks):
            if i >= len(old) or old[i] != blk:
                n += 1
                nbytes += blk[1]
    return n, nbytes


def expected_ring_bytes(table_base, table_now, second_now: set, bb: int) -> int:
    """Bytes an incremental snapshot must write itself: the blocks whose (hash, length) no block of the base has."""
    have = {blk for blocks in _blocks(table_base, bb).values() for blk in blocks} if table_base else set()
    return sum(blk[1] for rel, blocks in _blocks(table_now, bb).items() if rel not in second_now
               for blk in blocks if blk not in have)


def expected_pruned(man_dst: dict, man_src: dict) -> int:
    """Entries VMIG_F_PRUNE removes: in the destination, and the source has nothing of the same sort (directory or
    not) at that path."""
    isdir = lambda r: stat.S_ISDIR(r["type"])
    return sum(1 for rel, r in man_dst.items() if rel != "." and (rel not in man_src or isdir(man_src[rel]) != isdir(r)))
