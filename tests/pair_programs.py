"""Hand-written device programs aimed at the branches of `csrc/sbn_pair.cu` (TEST INFRASTRUCTURE).

The paired steps (`sbn_pair_kernel<M1, M2>`) and the expanding product (`sbn_triple_kernel`) are
mostly host-side decisions: how `spec_step` splits a step's tables into a main array and a per-row
`pre` factor, which evidence columns a canonical array gathers, which untouched axes a table
carries, how 4-state variables are padded.  A network search reaches few of them (the corpus's
`OPEN` list), but the engine runs any program words, so the programs here are written by hand.

A case is plain data:

    card   : variable -> cardinality (evidence columns included: their default card)
    ev     : the evidence columns, in column order
    tables : name -> "v0 v1 ..." or ("v0 v1 ...", {ev column: card of that axis in this table},
             {variable: state whose slice is all zero})
    steps  : (kind, output name, "inputs", "eliminated", "output axes, axis 0 first")
    slots  : output name -> slot, for the factors that must share a buffer (default: one each)

In a kind-1 step, an evidence column among an input's variables is gathered per row (a CPT's
evidence axis); in a kind-0 step it is an ordinary axis, so a kind-0 output can carry it to a
later gather.  `build` fills `planner.Plan` / `Step` / `_Factor` and serialises them with the
planner's own writer.  Table entries are float32 values in [0.25, 1] with about 15 % structural
zeros, so the float64 blob and the device's float32 blob hold the same numbers.

`branch` names the `sbn_pair.cu` code path a case is built for; `roles` is what
`Program.step_roles()` must report (None: not pinned) and `census` the `kernel_census.variants`
item its launch must show (None: no paired or triple launch).  Steps after the pair sum the
untouched axes out one at a time (5-term sums), which keeps the posterior small: a float32
normaliser over hundreds of entries alone would use up the 1e-6 budget.
"""
from __future__ import annotations

import itertools
from types import SimpleNamespace

import numpy as np

from sorobn_b200 import planner

T = 5  # SBN_PAIR_T
PAIR_SMEM_MAX = 40 * 1024  # SBN_PAIR_SMEM_MAX
PAIR_ROWS = 256  # SBN_PAIR_ROWS


def _dense_strides(cards):
    out, s = [], 1
    for c in cards:
        out.append(s)
        s *= c
    return out


def _values(cards, rng, zero=None, axes=()):
    """float32-representable entries in [0.25, 1], ~15 % zeros; `zero` = {axis name: state} zeroes
    that slice.  Flat, axis 0 fastest."""
    n = int(np.prod(cards, dtype=np.int64))
    v = rng.uniform(0.25, 1.0, n).astype(np.float32).astype(np.float64)
    v[rng.random(n) < 0.15] = 0.0
    arr = v.reshape(tuple(reversed(cards)))  # C order over reversed axes == axis 0 fastest
    for name, state in (zero or {}).items():
        k = axes.index(name)
        idx = [slice(None)] * len(cards)
        idx[len(cards) - 1 - k] = state
        arr[tuple(idx)] = 0.0
    return arr.reshape(-1)


def build(case, seed=0):
    """The program of a case: SimpleNamespace(plan, tables, ev, out_vars)."""
    rng = np.random.default_rng(seed)
    card, evcols = case["card"], list(case.get("ev", ()))
    var_id = {v: i for i, v in enumerate(card)}
    factors = {}  # name -> dict(vars, cards, strides, is_slot, buf, batched)
    arrays, tables = [], {}
    for t, spec in case["tables"].items():
        vs, over, zero = (spec, {}, {}) if isinstance(spec, str) else (tuple(spec) + ({}, {}))[:3]
        vs = tuple(vs.split())
        cards = tuple(over.get(v, card[v]) for v in vs)
        tables[t] = (vs, cards, _values(cards, rng, zero, vs))
        factors[t] = dict(vars=vs, cards=cards, strides=_dense_strides(cards), is_slot=False, buf=len(arrays), batched=False)
        arrays.append(tables[t][2])

    slot_of = dict(case.get("slots", {}))
    n_slots = max(slot_of.values(), default=-1) + 1
    slots = {}  # slot -> [batched, size]
    steps = []
    for kind, out, ins, elim, outv in case["steps"]:
        ins, elim, outv = ins.split(), tuple(elim.split()), tuple(outv.split())
        cards_of = {}
        inputs = []
        for name in ins:
            f = factors[name]
            stride = dict(zip(f["vars"], f["strides"]))
            ev = []
            for v, c in zip(f["vars"], f["cards"]):
                if kind == planner.KIND_BATCHED and v in evcols:
                    ev.append((evcols.index(v), stride[v], c))
                    continue
                assert v in elim or v in outv, (case["name"], name, v)
                assert cards_of.setdefault(v, c) == c, (case["name"], v)
            es = tuple(stride.get(v, 0) for v in elim)
            ss = tuple(stride.get(v, 0) for v in outv)
            fac = planner._Factor(f["is_slot"], f["buf"], tuple(var_id[v] for v in f["vars"]), tuple(f["strides"]),
                                  tuple(ev), f["batched"])
            inputs.append((fac, es, ss))
        ocards = tuple(cards_of[v] for v in outv)
        if out not in slot_of:
            slot_of[out] = n_slots
            n_slots += 1
        slot = slot_of[out]
        size = int(np.prod(ocards, dtype=np.int64))
        batched = kind == planner.KIND_BATCHED
        prev = slots.setdefault(slot, [batched, size])
        assert prev[0] == batched, (case["name"], out)
        prev[1] = max(prev[1], size)
        factors[out] = dict(vars=outv, cards=ocards, strides=_dense_strides(ocards), is_slot=True, buf=slot, batched=batched)
        steps.append(planner.Step(kind=kind, inputs=inputs, out_id=len(steps), out_vars=tuple(var_id[v] for v in outv),
                                  cards=ocards, elims=tuple(var_id[v] for v in elim),
                                  ecards=tuple(cards_of[v] for v in elim), out_slot=slot))
    last = factors[case["steps"][-1][1]]
    plan = planner.Plan(mode=planner.MODE_BATCHED, query=(), evidence=tuple(range(len(evcols))), order=[],
                        tables=list(range(len(arrays))), slots=[(bool(slots[s][0]), int(slots[s][1])) for s in range(n_slots)],
                        steps=steps, post_slot=last["buf"], Q=int(np.prod(last["cards"], dtype=np.int64)))
    planner._serialise(plan, arrays)
    return SimpleNamespace(plan=plan, tables=tables, ev=evcols, card=card, out_vars=last["vars"])


def ev_cards(built):
    """Largest card of each evidence column over the tables that gather it."""
    out = []
    for col in built.ev:
        cs = [c for vs, cards, _ in built.tables.values() for v, c in zip(vs, cards) if v == col]
        out.append(max(cs))
    return out


def evidence_rows(built, n_rows, seed=0):
    """uint8 codes [n_ev, n_rows]: the joint codes of every column over 0 .. card - 1, card and 255
    (codes at and above a table's card - 1 are clamped to it), shuffled, then repeated."""
    cards = ev_cards(built)
    if not cards:
        return np.zeros((0, n_rows), dtype=np.uint8)
    sets = [list(range(c)) + [c, 255] for c in cards]
    rng = np.random.default_rng(seed)
    if np.prod([len(s) for s in sets], dtype=np.float64) <= 4096:
        joint = np.array(list(itertools.product(*sets)), dtype=np.uint8).T
        joint = joint[:, rng.permutation(joint.shape[1])]
    else:
        joint = np.stack([rng.choice(s, 4096) for s in sets]).astype(np.uint8)
    reps = -(-n_rows // joint.shape[1])
    return np.ascontiguousarray(np.tile(joint, reps)[:, :n_rows])


def einsum_posterior(built, codes):
    """The normalised posterior [Q, B] and the totals [B] of the whole factor graph, by a direct
    float64 `np.einsum` per row: every table gathered at the row's (clamped) evidence codes, every
    variable that is not an output axis summed out."""
    letters = {v: chr(ord("a") + i) for i, v in enumerate(built.card)}
    out_sub = "".join(letters[v] for v in built.out_vars)
    B = codes.shape[1]
    post = np.zeros((built.plan.Q, B))
    for b in range(B):
        ops, subs = [], []
        for vs, cards, flat in built.tables.values():
            arr = flat.reshape(tuple(reversed(cards))).transpose()  # [v0, v1, ...]
            idx, sub = [], ""
            for v, c in zip(vs, cards):
                if v in built.ev:
                    idx.append(min(int(codes[built.ev.index(v), b]), c - 1))
                else:
                    idx.append(slice(None))
                    sub += letters[v]
            ops.append(arr[tuple(idx)])
            subs.append(sub)
        res = np.einsum(",".join(subs) + "->" + out_sub, *ops, optimize=True)
        post[:, b] = res.transpose().reshape(-1)  # axis 0 fastest
    total = post.sum(axis=0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return post / total, total


def unique_rows(codes):
    """(distinct columns, inverse): rows repeat, and the interpreter only needs each once."""
    if codes.shape[0] == 0:
        return codes[:, :1], np.zeros(codes.shape[1], dtype=np.int64)
    uniq, inv = np.unique(codes, axis=1, return_inverse=True)
    return np.ascontiguousarray(uniq), inv.reshape(-1)


# ---------------------------------------------------------------------------------------------------
# What sbn_pair_plan / plan_triple require of the words (the word-level preconditions)

def _axis_of_stride(cards, stride):
    acc = 1
    for j, c in enumerate(cards):
        if acc == stride and c > 1:
            return j
        acc *= c
    return -1


def tiled(st):
    """plan_tiles (sbn_api.cu) gives the step a tile: the inputs sorted by the tile axes they carry."""
    if st["kind"] != 1 or len(st["inputs"]) > 4:
        return False
    n_axes = len(st["cards"])
    us, as_, bs, cs = [], [], [], []
    for i, inp in enumerate(st["inputs"]):
        h0 = n_axes > 0 and inp["strides"][0] != 0
        h1 = n_axes > 1 and inp["strides"][1] != 0
        (cs if h0 and h1 else as_ if h0 else bs if h1 else us).append(i)
    if len(cs) > 1:
        return False
    if not cs:
        while len(us) > 2 or (not as_ and us):
            if len(as_) < 2:
                as_.append(us.pop())
            elif n_axes > 1 and len(bs) < 2:
                bs.append(us.pop())
            else:
                break
        return not (len(us) > 2 or not as_ or len(as_) > 2 or len(bs) > 2 or (n_axes > 1 and not bs))
    return len(us) <= 1 and len(as_) <= 1 and len(bs) <= 1


def pair_conditions(words, i1, i2, slot_sizes):
    """The conditions of sbn_pair_plan on steps i1, i2 (as named booleans)."""
    from oracle import program_interp

    hdr, _, _, steps = program_interp.parse(words)
    s1, s2 = steps[i1], steps[i2]
    c = {"kinds": s1["kind"] == 1 and s2["kind"] == 1 and len(s1["ecards"]) == 1 and len(s2["ecards"]) == 1}
    c["tiled"] = tiled(s1) and tiled(s2)
    b1 = [i for i, inp in enumerate(s1["inputs"]) if inp["batched"]]
    b2 = [i for i, inp in enumerate(s2["inputs"]) if inp["batched"]]
    c["batched operands"] = len(b1) in (1, 2) and len(b2) == 1
    if not (c["kinds"] and c["batched operands"]):
        return c
    M = s2["inputs"][b2[0]]
    c["mid is step 1's output"] = M["is_slot"] == 1 and M["buf"] == s1["out_slot"] and not M["ev"]
    jy = _axis_of_stride(s1["cards"], M["estrides"][0])
    fi, gi = b1[-1], (b1[0] if len(b1) == 2 else -1)
    if gi >= 0:
        F, G = s1["inputs"][fi], s1["inputs"][gi]
        if F["strides"][jy] == 0 or (G["strides"][jy] != 0 and slot_sizes[G["buf"]] > slot_sizes[F["buf"]]):
            fi, gi = gi, fi
        c["G apart from step 2's output"] = s1["inputs"][gi]["buf"] != s2["out_slot"]
        c["no tables beside G"] = len(s1["inputs"]) == 2
    F = s1["inputs"][fi]
    c["F apart from step 2's output"] = F["buf"] != s2["out_slot"]
    c["step 1's output is not the posterior"] = s1["out_slot"] != hdr["post_slot"]
    c["F carries y"] = jy >= 0 and F["strides"][jy] != 0 and not F["ev"]
    # out2 -> out1 axes, exactly one new variable z, and a variable w that step 1 introduces
    new = [k for k in range(len(s2["cards"])) if M["strides"][k] == 0]
    to1 = {k: _axis_of_stride(s1["cards"], M["strides"][k]) for k in range(len(s2["cards"])) if k not in new}
    c["one new variable z"] = len(new) == 1 and len(s2["cards"]) == len(s1["cards"]) and all(
        j >= 0 and j != jy and s1["cards"][j] == s2["cards"][k] for k, j in to1.items())
    ws = [k for k, j in to1.items() if F["strides"][j] == 0]
    cards = [s1["ecards"][0], s2["ecards"][0]] + ([s2["cards"][new[0]]] if new else []) + [s2["cards"][k] for k in ws[:1]]
    c["cardinalities 4 or 5"] = len(ws) >= 1 and all(4 <= x <= T for x in cards) and (gi < 0 or all(x == T for x in cards))
    return c


def triple_conditions(words, i1, i2):
    """The conditions of plan_triple on steps i1, i2 that the words show directly."""
    from oracle import program_interp

    hdr, _, _, steps = program_interp.parse(words)
    s1, s2 = steps[i1], steps[i2]
    c = {"kinds": s1["kind"] == 1 and s2["kind"] == 1 and len(s1["ecards"]) == 1 and len(s2["ecards"]) == 2}
    c["two batched operands each"] = all(len(s["inputs"]) == 2 and all(i["batched"] and i["is_slot"] and not i["ev"] for i in s["inputs"])
                                         for s in (s1, s2))
    c["eliminated cards 5"] = list(s1["ecards"]) + list(s2["ecards"]) == [T, T, T]
    mids = [i for i in s2["inputs"] if i["buf"] == s1["out_slot"]]
    c["mid is one operand of step 2"] = len(mids) == 1
    c["step 1's output is not the posterior"] = s1["out_slot"] != hdr["post_slot"]
    c["output apart from the operands"] = all(i["buf"] != s2["out_slot"] for i in s1["inputs"] + s2["inputs"])
    return c


def multi_chunk_rows(n_tiles, n_sms):
    """Smallest row count at which sbn_pair_launch gives a CTA more than one tile and the last chunk
    fewer than the others (target 8 x SMs x 6 CTAs), or None."""
    target = 8 * n_sms * 6
    for n_rblocks in range(1, 1 << 12):
        chunks = max(1, min(n_tiles, target // n_rblocks))
        tpc = -(-n_tiles // chunks)
        if tpc > 1 and n_tiles % tpc:
            return (n_rblocks - 1) * PAIR_ROWS + 1
    return None


# ---------------------------------------------------------------------------------------------------
# The cases

_PAIR_CARD = dict(x=5, y=5, w=5, z=5, e0=3, e1=3, e2=4, e3=3)


def _pair(name, branch, tables1, tables2, census, card=None, r=(), extra_tables=None, pre_steps=(),
          g=None, slots=None, tail=None, roles=None, ev=("e0", "e1", "e2", "e3"), multi_chunk=None):
    """A pair program: F = S (per row, over x, y and the untouched axes r), then
    step 1: mid[y, w, r] = sum_x F x tables1 (x G when `g` names G's variables), and
    step 2: out[w, z, r] = sum_y mid x tables2; then the untouched axes are summed out one by one.
    `multi_chunk`: the pair's tile count, for a run at `multi_chunk_rows`."""
    card = {**_PAIR_CARD, **(card or {})}
    rs = " ".join(r)
    tables = {"S": (f"x y {rs} e0", {}, {"e0": 1})}  # rows with e0 = 1 are impossible
    tables.update(extra_tables or {})
    steps = list(pre_steps)
    steps.append((1, "F", "S", "", f"x y {rs}"))
    in1 = "F"
    if g is not None:
        # G first: of two batched operands of one size, sbn_pair_plan takes the last as F
        tables["SG"] = f"{g} e0"
        steps.append((1, "G", "SG", "", g))
        in1 = "G F"
    for k, v in enumerate(tables1):
        if isinstance(v, str) and v.startswith("@"):  # the output of an earlier step
            in1 += f" {v[1:]}"
            continue
        tables[f"T1{k}"] = v
        in1 += f" T1{k}"
    in2 = "M"
    for k, v in enumerate(tables2):
        tables[f"T2{k}"] = v
        in2 += f" T2{k}"
    steps.append((1, "M", in1, "x", f"y w {rs}"))
    steps.append((1, "O", in2, "y", f"w z {rs}"))
    left = ["w", "z", *r]
    prev = "O"
    for k, v in enumerate(r):
        left.remove(v)
        steps.append((1, f"R{k}", prev, v, " ".join(left)))
        prev = f"R{k}"
    steps += list(tail or ())
    used = {v for t in tables.values() for v in (t if isinstance(t, str) else t[0]).split()}
    n_pre = sum(1 for s in pre_steps if s[0] == 0)
    n_src = 1 + (g is not None)
    if roles is None and census is not None:
        roles = [0] * n_pre + [1] * n_src + [2, 3] + [1] * (len(r) + len(tail or ()))
    return dict(name=name, branch=branch, card={k: v for k, v in card.items() if k in used or k in ("x", "y", "w", "z")},
                ev=[e for e in ev if e in used], tables=tables, steps=steps, slots=slots or {}, census=census, roles=roles,
                pair=(n_pre + n_src, n_pre + n_src + 1), multi_chunk=multi_chunk)


def _triple(name, branch, a, b, c, mid, out, group, card=None, tail=()):
    """A triple program: A, B, C per row (each from a table over its variables and e0), then
    step 1: mid = sum_j A x B (an expanding product), step 2: out = sum_{p, k} mid x C, then `tail`."""
    card = {**dict(j=5, k=5, p=5, s=5, z=5, e0=3, e1=4), **(card or {})}
    tables = {"SA": (f"{a} e0", {}, {"e0": 1}), "SB": f"{b} e1", "SC": f"{c} e0"}
    steps = [(1, "A", "SA", "", a), (1, "B", "SB", "", b), (1, "C", "SC", "", c),
             (1, "M", "A B", "j", mid), (1, "O", "M C", "p k", out), *tail]
    return dict(name=name, branch=branch, card=card, ev=["e0", "e1"], tables=tables, steps=steps, slots={},
                census=f"triple group={group}", roles=[1, 1, 1, 4, 5] + [1] * len(tail), pair=(3, 4), multi_chunk=None)


PAIR_CASES = [
    # ---- the 15 (m1, m2) mode pairs; spec_step picks the layout from the tables each step multiplies
    _pair("B_B_pre1_pre2", "m1 = B (no main table carries y), m2 = B; has_pre1 (E over x, y, e1) and has_pre2 (E over y, w, e2) "
          "together", ["x w", "x y e1"], ["y z", "y w e2"], "pair (0,0)"),
    _pair("B_CU_ev1_y4", "m1 = B with one evidence column in the main array (main_ev without main_d0), m2 = CU; y at 4 states",
          ["x w e1"], ["y w z"], "pair (0,1)", card=dict(y=4)),
    _pair("B_CE_ev2_z4", "m1 = B, m2 = CE gathering two columns; z at 4 states", ["x w"], ["y w z e1 e2"], "pair (0,2)",
          card=dict(z=4)),
    _pair("CU_B_pre1_w4", "m1 = CU with has_pre1 alone (E over x, e1 leaves the main array), m2 = B; w at 4 states",
          ["x y w", "x e1"], ["y z"], "pair (1,0)", card=dict(w=4)),
    _pair("CU_CU_r1", "m1 = CU, m2 = CU with has_pre2 (E over y, e1); one untouched axis r0 that both main tables carry "
          "(r_axes, tile_slab)", ["x y w r0"], ["y w z r0", "y e1"], "pair (1,1)", card=dict(r0=3), r=("r0",)),
    _pair("CU_CE_pre1", "m1 = CU with has_pre1 (E over x, y absent, e2), beside a CE main array in step 2",
          ["x y w", "x e2"], ["y w z e1"], "pair (1,2)"),
    _pair("CE_B_pre2", "m1 = CE (one table over x, y, w, e1), m2 = B with has_pre2 alone (E over y, w, e2)",
          ["x y w e1"], ["y z", "y w e2"], "pair (2,0)"),
    _pair("CE_CU_merge_x4", "m1 = CE: a table over x, w and two columns joins a table over x, y, w in the main array "
          "(main_ev and main_d0: no pre), m2 = CU; x at 4 states", ["x y w", "x w e1 e2"], ["y w z"], "pair (2,1)",
          card=dict(x=4)),
    _pair("CE_CE_ev3_shared", "m1 = CE gathering three columns, m2 = CE whose two tables share column e1 at cards 5 and 3 "
          "(size_canon keeps the larger, fill_canon clamps per table)", ["x y w e1 e2 e3"],
          [("y w z e1", {"e1": 5}), ("y z e1", {"e1": 3})], "pair (2,2)", card=dict(e2=2, e3=2)),
    _pair("GB_B", "m1 = GB: a second batched operand G over x, w (no tables, all cards 5), m2 = B with has_pre2",
          [], ["y z", "y w e2"], "pair (3,0)", g="x w"),
    _pair("GB_CU", "m1 = GB, m2 = CU", [], ["y w z"], "pair (3,1)", g="x w"),
    _pair("GB_CE", "m1 = GB, m2 = CE", [], ["y w z e1"], "pair (3,2)", g="x w"),
    _pair("GC_B", "m1 = GC: G over x, y, w; F carries an untouched axis r0 (5 states) so it is not smaller than G", [], ["y z"],
          "pair (4,0)", g="x y w", card=dict(r0=5), r=("r0",)),
    _pair("GC_CU", "m1 = GC, m2 = CU", [], ["y w z"], "pair (4,1)", g="x y w", card=dict(r0=5), r=("r0",)),
    _pair("GC_CE", "m1 = GC, m2 = CE gathering two columns", [], ["y w z e1 e2"], "pair (4,2)", g="x y w", card=dict(r0=5),
          r=("r0",)),
    # ---- padding, evidence gathers, untouched axes, table steps
    _pair("CU_CE_all4", "x, y, w and z all at 4 states (the 5 x 5 x 5 loop nest zero-padded on every axis), m1 = CU with "
          "has_pre1, m2 = CE", ["x y w", "x e1"], ["y w z e2"], "pair (1,2)", card=dict(x=4, y=4, w=4, z=4)),
    _pair("B_CE_ev4", "m2 = CE gathering four columns (SBN_PAIR_MAX_EV), m1 = B gathering none", ["x w"],
          ["y w z e0 e1 e2 e3"], "pair (0,2)", card=dict(e0=2, e1=3, e2=2, e3=3)),
    _pair("CU_CU_r3", "three untouched axes: r0, r1 in step 1's main array, r2 in step 2's (each canonical array carries its "
          "own subset: tile_slab maps the digits)", ["x y w r0 r1"], ["y w z r2"], "pair (1,1)",
          card=dict(r0=2, r1=3, r2=2), r=("r0", "r1", "r2")),
    _pair("B_table_step", "step 1's main table is the unbatched output of a kind-0 step (host_table's slot branch), no "
          "evidence axes", ["@K"], ["y w z"], "pair (0,1)", card=dict(u=3),
          extra_tables={"Ka": "u x", "Kb": "u w"}, pre_steps=[(0, "K", "Ka Kb", "u", "x w")]),
    _pair("B_table_step_ev", "step 1's main table is a kind-0 output that carries evidence column e1 as an axis, gathered "
          "per row by the pair (host_table's slot branch with an evidence axis)", ["@K"], ["y z"], "pair (0,0)",
          card=dict(u=3), extra_tables={"Ka": "u x e1", "Kb": "u w"}, pre_steps=[(0, "K", "Ka Kb", "u", "x w e1")]),
    _pair("smem_just_under", "canonical arrays of 40,880 B: B over e1 (5 states, 220 floats) + CE over e2, e3 (8 x 10, "
          "10,000 floats), just under SBN_PAIR_SMEM_MAX", [("x w e1", {"e1": 5})], [("y w z e2 e3", {"e2": 8, "e3": 10})],
          "pair (0,2)"),
    _pair("smem_just_over", "the same with e1 at 6 states: 41,056 B, over SBN_PAIR_SMEM_MAX (each array alone fits): "
          "single-step launches", [("x w e1", {"e1": 6})], [("y w z e2 e3", {"e2": 8, "e3": 10})], None,
          roles=[1, 1, 1]),
    _pair("card1_axis", "an untouched axis of one state (axis_of_stride skips it): pairing or not, the result must hold",
          ["x y w r0"], ["y w z r0"], None, card=dict(r0=1), r=("r0",), roles=None),
    # ---- refusals: both must run as single steps
    _pair("refuse_F_is_out2", "F's slot is step 2's output slot: the launch would overwrite F while reading it",
          ["x y w"], ["y w z"], None, slots={"F": 0, "O": 0}, roles=[1, 1, 1]),
    _pair("refuse_out1_is_post", "step 1 writes the posterior slot (a later step re-uses it): refused",
          ["x y w"], ["y w z"], None, slots={"F": 0, "M": 1, "P": 1}, tail=[(1, "P", "O", "", "w z")], roles=[1, 1, 1, 1]),
    # ---- launch geometry: 125 tiles per row block, more rows than 8 x SMs x 6 CTAs cover at one tile each
    _pair("CU_CU_multi_chunk", "125 tiles (three 5-state untouched axes): sbn_pair_launch's tiles_per_cta > 1 with a partial "
          "last chunk at the multi-chunk row count", ["x y w r0"], ["y w z"], "pair (1,1)", card=dict(r0=5, r1=5, r2=5),
          r=("r0", "r1", "r2"), multi_chunk=125),
]

TRIPLE_CASES = [
    _triple("triple_g5_r0", "group 5: g (5 states) is a tile axis only A carries; no other untouched axis",
            "g p k j", "p j s", "k z p", "g p k s", "g z s", 5, card=dict(g=5),
            tail=[(1, "R", "O", "g", "z s")]),
    _triple("triple_g5_r1", "group 5 with one untouched axis q (3 states) carried by B and C",
            "g p k j", "p q j s", "k q z p", "g p k s q", "g z s q", 5, card=dict(g=5, q=3),
            tail=[(1, "R", "O", "g", "z s q"), (1, "R2", "R", "q", "z s")]),
    _triple("triple_g5_r2", "group 5 with two untouched axes: a (3 states, A only) and q (2 states, B and C)",
            "a g p k j", "p q j s", "k q z p", "a g p k s q", "a g z s q", 5, card=dict(g=5, a=3, q=2),
            tail=[(1, "R", "O", "g", "a z s q"), (1, "R2", "R", "a", "z s q"), (1, "R3", "R2", "q", "z s")]),
    _triple("triple_g1_r0", "group 1: no axis only A carries, no untouched axis (one tile, 128 x 1 CTAs)",
            "p k j", "p j s", "k z p", "p k s", "z s", 1),
    _triple("triple_g1_a4", "group 1: the axis only A carries has 4 states, so it is an untouched tile axis",
            "a p k j", "p j s", "k z p", "a p k s", "a z s", 1, card=dict(a=4),
            tail=[(1, "R", "O", "a", "z s")]),
    _triple("triple_g1_r2", "group 1 with two untouched axes: a (4 states, A only) and q (3 states, B and C)",
            "a p k j", "p q j s", "k q z p", "a p k s q", "a z s q", 1, card=dict(a=4, q=3),
            tail=[(1, "R", "O", "a", "z s q"), (1, "R2", "R", "q", "z s")]),
]

CASES = PAIR_CASES + TRIPLE_CASES


def case_id(case):
    return case["name"]
