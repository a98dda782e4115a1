"""CPU checks of the DV <= 64 attention schedule in powerpaint_b200/csrc/attention.cu: tensor-core turns between the
two consumer warpgroups and the look-ahead of one key block.

Per key block j a consumer warp of warpgroup g waits for `kv_full` of block j + 1, takes its turn (named barrier
1 + g), issues S(j+1) = Q K(j+1)^T and O += P(j) V(j), hands the turn over (named barrier 2 - g), waits for S(j+1),
then for PV(j), and only then releases stage j on `kv_empty`. So a warp holds two ring stages at once. The model below
restates that program for G = 2 warpgroups of W warps, next to the producer of test_attention_protocol_model.py, and
explores every interleaving for small key counts, checking:

  TMA load issued    -> no warp still needs the block the stage held (its last MMA on it has not retired)
  MMA issued on j    -> the stage holds key block j, completely landed
  MMA issued         -> the other warpgroup is not inside its turn
  end of every run   -> all warps and the producer are done, and no named barrier holds pending arrivals

A named barrier of 256 threads is (completed generations, arrived warps): bar.arrive adds a warp, bar.sync adds one and
waits for the generation it joined to complete. Mutants show the model sees what it is meant to exclude.
The compiled-code tests read what `build()` left: the look-ahead must keep S(j+1) in flight past a
`WARPGROUP.DEPBAR.LE gsb0, 0x1`, and no variant up to DV = 128 may spill or have its wgmma serialised.
"""
import os
import re
import subprocess
from collections import deque
from pathlib import Path

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(os.path.dirname(HERE), "powerpaint_b200", "csrc", "attention.cu")


class Violation(Exception):
    pass


def program(g, nkv, mutant=None):
    """the op list every warp of warpgroup g runs (attn_fwd_kernel, DCH == 1 consumer branch)"""
    mine, other = ("T0", "T1") if g == 0 else ("T1", "T0")
    ops = [("arrive", other)] if g == 1 else []
    ops += [("wait_q",), ("wait_full", 0), ("sync", mine), ("issue", ("S", 0)), ("arrive", other),
            ("retire", None)]
    for j in range(nkv - 1):
        body = [("wait_full", j + 1), ("sync", mine), ("issue", ("S", j + 1)), ("issue", ("PV", j)),
                ("arrive", other), ("retire", None), ("retire", j), ("release", j)]
        if mutant == "early_release":
            body.remove(("release", j))
            body.insert(body.index(("arrive", other)) + 1, ("release", j))
        ops += body
    ops += [("sync", mine), ("issue", ("PV", nkv - 1))]
    if g == 0 and mutant != "missing_handover":
        ops += [("arrive", other)]
    if g == 1 and mutant == "extra_handover":
        ops += [("arrive", other)]
    ops += [("retire", nkv - 1), ("release", nkv - 1)]
    if mutant == "no_turns":
        ops = [op for op in ops if op[0] not in ("sync", "arrive")]
    return ops


def explore(nkv, S, W, mutant=None, max_states=5_000_000):
    """all interleavings of the producer and 2 x W consumer warps; returns the number of distinct states"""
    G = 2
    progs = [program(g, nkv, mutant) for g in range(G)]
    # A batch is a run of consecutive issues (one turn). Per pc: batches begun, batches completed, and the last block
    # whose final MMA has retired.
    begun, completed, done = [], [], []
    for ops in progs:
        bg, cp, dn, nb, last = [], [], [], 0, -1
        for k, op in enumerate(ops):
            bg.append(nb)
            cp.append(nb - (k > 0 and ops[k - 1][0] == "issue" and op[0] == "issue"))
            dn.append(last)
            if op[0] == "issue" and (k == 0 or ops[k - 1][0] != "issue"):
                nb += 1
            if op[0] == "retire" and op[1] is not None:
                last = op[1]
        bg.append(nb)
        cp.append(nb)
        dn.append(last)
        begun.append(bg)
        completed.append(cp)
        done.append(dn)
    nwarps = G * W
    # state: q landed, producer next block, full[s] phases, empty[s] (phases, pending), stage[s] = (block, landed),
    # turn barriers {T0, T1} as (generations, pending), warps per group as sorted tuples of (pc, generation joined)
    init = (False, 0, (0,) * S, ((0, 0),) * S, ((-1, True),) * S, ((0, 0), (0, 0)),
            tuple(tuple((0, -1) for _ in range(W)) for _ in range(G)))
    seen = {init}
    todo = deque([init])
    tid = {"T0": 0, "T1": 1}

    def passed(phases, parity):
        return (phases & 1) != parity

    while todo:
        st = todo.popleft()
        q, pj, full, empty, stage, turns, warps = st
        succ = []
        if not q:
            succ.append((True, pj, full, empty, stage, turns, warps))
        elif pj < nkv:
            s = pj % S
            if passed(empty[s][0], ((pj // S) & 1) ^ 1):
                old = stage[s][0]
                for g in range(G):
                    if old >= 0 and any(done[g][pc] < old for pc, _ in warps[g]):
                        raise Violation(f"stage {s}: TMA load of block {pj} overwrites block {old} under a reader")
                succ.append((q, pj + 1, full, empty, stage[:s] + ((pj, False),) + stage[s + 1:], turns, warps))
        for s, (blk, landed) in enumerate(stage):
            if not landed:
                succ.append((q, pj, full[:s] + (full[s] + 1,) + full[s + 1:], empty,
                             stage[:s] + ((blk, True),) + stage[s + 1:], turns, warps))
        for g in range(G):
            for i, (pc, joined) in enumerate(warps[g]):
                if i > 0 and warps[g][i - 1] == (pc, joined):
                    continue
                ops = progs[g]
                if pc >= len(ops):
                    continue
                op = ops[pc]

                def moved(pc2, joined2=-1, turns2=turns, full2=full, empty2=empty):
                    rest = warps[g][:i] + warps[g][i + 1:]
                    w2 = tuple(sorted(rest + ((pc2, joined2),)))
                    return (q, pj, full2, empty2, stage, turns2, warps[:g] + (w2,) + warps[g + 1:])

                if op[0] == "wait_q":
                    if q:
                        succ.append(moved(pc + 1))
                elif op[0] == "wait_full":
                    j = op[1]
                    if passed(full[j % S], (j // S) & 1):
                        succ.append(moved(pc + 1))
                elif op[0] in ("arrive", "sync"):
                    t = tid[op[1]]
                    gen, pend = turns[t]
                    if op[0] == "sync" and joined >= 0:
                        if gen > joined:
                            succ.append(moved(pc + 1))
                        continue
                    pend += 1
                    if pend == nwarps:
                        gen, pend = gen + 1, 0
                    turns2 = turns[:t] + ((gen, pend),) + turns[t + 1:]
                    if op[0] == "arrive":
                        succ.append(moved(pc + 1, turns2=turns2))
                    else:
                        succ.append(moved(pc, turns[t][0], turns2=turns2))
                elif op[0] == "issue":
                    kind, j = op[1]
                    if stage[j % S] != (j, True):
                        raise Violation(f"stage {j % S}: a warp issues {kind}({j}) but the stage holds {stage[j % S]}")
                    # turns alternate, warpgroup 0 first: its batch k follows the other's batch k - 1, warpgroup 1's
                    # batch k follows the other's batch k
                    k = begun[g][pc] - (pc > 0 and ops[pc - 1][0] == "issue")
                    lo = k + g
                    if any(completed[1 - g][pc2] < lo or begun[1 - g][pc2] > lo for pc2, _ in warps[1 - g]):
                        raise Violation(f"warpgroup {g} issues {kind}({j}) out of turn")
                    succ.append(moved(pc + 1))
                elif op[0] == "retire":
                    succ.append(moved(pc + 1))
                elif op[0] == "release":
                    s = op[1] % S
                    c, pnd = empty[s]
                    pnd += 1
                    if pnd == nwarps:
                        c, pnd = c + 1, 0
                    succ.append(moved(pc + 1, empty2=empty[:s] + ((c, pnd),) + empty[s + 1:]))
        if not succ:
            finished = all(pc >= len(progs[g]) for g in range(G) for pc, _ in warps[g])
            if not (finished and pj == nkv and all(ld for _, ld in stage)):
                raise Violation(f"deadlock in state {st}")
            if any(pend for _, pend in turns):
                raise Violation(f"a turn barrier is left with pending arrivals: {turns}")
        for n in succ:
            if n not in seen:
                seen.add(n)
                todo.append(n)
                if len(seen) > max_states:
                    raise RuntimeError("state space larger than expected")
    return len(seen)


@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("nkv", [1, 2, 3, 4, 5, 6])
def test_every_interleaving_of_the_look_ahead_schedule(nkv, S):
    assert explore(nkv, S, W=2) > 10


@pytest.mark.parametrize("nkv,S", [(1, 3), (2, 3), (3, 2)])
def test_four_warps_per_warpgroup(nkv, S):
    """the kernel's 2 x 4 consumer warps, key counts small enough to stay quick"""
    assert explore(nkv, S, W=4) > 10


def test_an_early_release_is_visible_to_the_model():
    """releasing stage j before PV(j) has retired lets the producer refill it under the MMA"""
    with pytest.raises(Violation, match="under a reader"):
        explore(4, 2, 2, mutant="early_release")


def test_a_single_stage_ring_deadlocks_with_look_ahead():
    """a warp holds stage j + 1 before it releases stage j: one stage cannot serve that"""
    with pytest.raises(Violation, match="deadlock"):
        explore(3, 1, 2)


def test_a_missing_hand_over_is_visible_to_the_model():
    """warpgroup 0 does not hand the last turn over: warpgroup 1 waits forever"""
    with pytest.raises(Violation, match="deadlock"):
        explore(2, 2, 2, mutant="missing_handover")


def test_a_hand_over_too_many_leaves_a_barrier_pending():
    with pytest.raises(Violation, match="pending"):
        explore(2, 2, 2, mutant="extra_handover")


def test_without_turns_the_warpgroups_issue_together():
    with pytest.raises(Violation, match="turn"):
        explore(2, 2, 2, mutant="no_turns")


def test_model_matches_the_source():
    """the turns, waits and releases the model restates, verbatim in attention.cu and in the model's order"""
    src = open(SRC).read()
    start = src.index("} else if constexpr (DCH == 1) {")
    body = src[start:src.index("// epilogue", start)]
    for line in [
        'static_assert(S >= 2, "the look-ahead holds two ring stages at once");',
        "const int turn_mine = 1 + wg, turn_other = 2 - wg;",
        "if (wg == 1) named_bar_arrive(turn_other, 256);  // warpgroup 0 takes the first turn",
        "if (wg == 0) named_bar_arrive(turn_other, 256);  // the last turn is warpgroup 1's: nothing left pending",
    ]:
        assert line in body, f"attention.cu no longer contains `{line}`: update the schedule model"
    loop = body[body.index("for (int j = 0; j + 1 < nkv; ++j) {"):]
    order = ["mbar_wait(bar_kv_full(s1), ((j + 1) / S) & 1);", "named_bar_sync(turn_mine, 256);", "issue_s(j + 1);",
             "issue_pv(j);", "named_bar_arrive(turn_other, 256);", "wgmma_wait<1>();", "wgmma_wait<0>();",
             "if (lane == 0) mbar_arrive(bar_kv_empty(s));"]
    pos = [loop.index(x) for x in order]
    assert pos == sorted(pos), "the look-ahead loop no longer runs in the order the model restates"
    last = loop[loop.index("if (lane == 0) mbar_arrive(bar_kv_empty(s));"):]
    order = ["named_bar_sync(turn_mine, 256);", "issue_pv(nkv - 1);", "if (wg == 0) named_bar_arrive",
             "wgmma_wait<0>();", "if (lane == 0) mbar_arrive(bar_kv_empty(s));"]
    pos = [last.index(x, 1) for x in order]
    assert pos == sorted(pos), "the last block no longer runs in the order the model restates"


# --------------------------------------------------------------------------- compiled code
ATTN = re.compile(r"_ZN2pp15attn_fwd_kernelILi(\d+)ELb([01])EEEvNS_11AttnKParamsE")


@pytest.fixture(scope="module")
def built():
    from powerpaint_b200 import build as b

    b.build()
    stem = b.BUILD_DIR / "attention"
    nvcc = b._nvcc()
    import shutil

    cuobjdump = str(Path(shutil.which(nvcc) or nvcc).resolve().parent / "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", str(stem) + ".o"], capture_output=True, text=True, check=True).stdout
    return Path(str(stem) + ".ptxas.log").read_text(), sass


def test_look_ahead_keeps_one_mma_group_in_flight(built):
    """every DV <= 64 variant waits for S(j+1) alone (`DEPBAR.LE gsb0, 0x1`) and runs the 64 exponentials of the block
    before it waits for PV(j): ptxas moves such waits up unless the source pins the exponentials above them"""
    _, sass = built
    overlapped = {}  # function -> MUFU.EX2 between a `0x1` wait and the next wait
    fn, inside = None, False
    for line in sass.splitlines():
        m = re.search(r"Function : (\w+)", line)
        if m:
            fn, inside = m.group(1), False
            overlapped[fn] = 0
        elif fn and "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line:
            inside = True
        elif fn and "WARPGROUP.DEPBAR" in line:
            inside = False
        elif inside and "MUFU.EX2" in line:
            overlapped[fn] += 1
    look_ahead = {fn: n for fn, n in overlapped.items() if ATTN.match(fn) and int(ATTN.match(fn).group(1)) <= 64}
    assert len(look_ahead) == 6, sorted(look_ahead)
    assert all(n >= 64 for n in look_ahead.values()), f"exponentials overlapping PV(j): {look_ahead}"


def test_no_spill_and_no_serialised_wgmma_up_to_dv128(built):
    log, _ = built
    stats = {}
    for m in re.finditer(r"Compiling entry function '(\w+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         re.S):
        stats[m.group(1)] = int(m.group(2)) + int(m.group(3))
    checked = {fn: n for fn, n in stats.items() if ATTN.match(fn) and int(ATTN.match(fn).group(1)) <= 128}
    assert len(checked) == 12, sorted(checked)
    assert not any(checked.values()), f"spills: {checked}"
    warned = {fn for _, fn in re.findall(r"\((C75\d\d)\).*?function '(\w+)'", log) if fn in checked}
    assert not warned, f"ptxas serialised the wgmma of: {sorted(warned)}"
