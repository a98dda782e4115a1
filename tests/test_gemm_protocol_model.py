"""CPU model check of the hand-over protocol of the GEMM / conv kernel (gemm_conv_kernel, powerpaint_b200/csrc/gemm_conv.cu).

One CTA runs a TMA producer thread, W consumer warps (the kernel: 8, two warpgroups) and, in mode 3, a ticket-server
lane. Every role is restated below as a small program: a list of ops, one per wait, arrival, copy or access of shared
state the source makes, in the source's order and with the parity the source passes to each `mbar_wait`. One
interpreter (`thread_step` in `explore`) gives each op its meaning, and `explore` runs every interleaving of the programs and of the
asynchronous events (a TMA load or residual landing, a cp.async landing, a TMA store's "read done" and then its "global
write done", the other lanes of a warp finishing their statistics-pass reads) breadth-first. Threads of the same role
are interchangeable, so a state keeps them as a sorted tuple: the states are counted up to a permutation of the warps.

The resources and what the model requires of them (a breach raises `Violation` naming the resource):

  ring stage      a TMA load only when no unretired wgmma group reads the stage; a wgmma only on landed bytes of
                  its own k-iteration
  staging tile    a residual TMA write only when no TMA store still reads the tile and no warp (no lane) is still in
                  the previous tile's epilogue or statistics pass; the epilogue reads this tile's residual, landed;
                  a TMA store reads only after every warp's writes of the tile, their proxy fences and the barrier;
                  the statistics pass reads this tile's results; without a staged residual the epilogue writes
                  the tile only after the previous stores have read it
  bias/u buffer   buffer acc ^ 1 is written only after tile lt - 1's last read of it; tile lt reads its own values
  s_row           written only after the previous tile's statistics pass has read it
  split-K         the owner reads the workspace only after the donor's complete, published write; the flag is 0
                  at the end of the launch
  mode 3          a verdict read belongs to its own request; each row block is folded exactly once per warp slice,
                  after all of its records are written; row_ticket is 0 at the end of the launch
  progress        every run ends with all roles done, no barrier holding pending arrivals and nothing outstanding:
                  a thread that exits with a bulk group or a cp.async in flight is a violation

Conventions (as in test_attention_protocol_model.py / test_attention_schedule_cpu.py): an mbarrier is (completed
phases, pending arrivals) and `wait(parity)` passes iff the phase in progress has the other parity (PTX
`mbarrier.try_wait.parity`); a named barrier of the consumer warps is (completed generations, arrived warps), and
`bar.sync` joins the generation in progress and waits for it to complete. A wgmma group is a reader of its stage until
the `wgmma_wait` that retires it. Only `__syncwarp` and `bar.sync` order the shared-memory accesses of the lanes of a
warp (PTX: `shfl.sync`, `ldmatrix` / `stmatrix` and the `.aligned` wgmma do not): each warp's program is that of its
lane 0, and after the statistics pass the other lanes may still be reading until the warp's next `__syncwarp` or
`bar.sync`, or until they catch up on their own.

Two reduced models sit next to the CTA model: the split-K pair (owner and donor CTA, their hand-over through the
workspace and the flag; their rings are the CTA model's) and mode 3 across two or three CTAs (one epilogue warp and one
ticket server each, tiles dealt out as the kernel's walk deals them), so that exactly one CTA folds each row block.

`test_model_matches_the_source` ties the model to gemm_conv.cu: each line the programs restate is there verbatim, in
the order the programs assume, so an edit of the protocol fails here until the model follows it.
"""
import os
import re
import time
from collections import deque

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(os.path.dirname(HERE), "powerpaint_b200", "csrc", "gemm_conv.cu")

GEMM_EPI_WARPS = 8


class Violation(Exception):
    pass


# =========================================================================== programs
class Config:
    """one launch shape of the model: S ring stages, K k-iterations per tile, T tiles per CTA, W consumer warps of
    which `storers` issue a TMA store (lane 0 of warps 0 .. BLOCK_N / 64 - 1), MODE 0 / 1 / 3 / 5"""

    def __init__(self, S, K, T, mode, stage_res=False, stage_rv=False, W=2, storers=None, n_tiles=1, mutant=None,
                 bias=True):
        assert mode in (0, 1, 3, 5)
        assert not ((stage_res or stage_rv) and mode not in (0, 3)), "res1 / the row vector are staged in modes 0 / 3"
        self.S, self.K, self.T, self.mode, self.W = S, K, T, mode, W
        self.stage_res, self.stage_rv, self.mutant = stage_res, stage_rv, mutant
        # the next tile's bias / u row goes in by cp.async when the launch has a bias or a staged row vector (else the
        # top of the tile stores zeros)
        self.async_bias = bias or stage_rv
        self.storers = 0 if mode == 1 else (W if storers is None else storers)
        self.stats = mode in (0, 3)  # the GroupNorm statistics pass (p.chan_stats) reads the staging tile
        self.n_tiles = n_tiles
        self.tiles = [(t // n_tiles, t % n_tiles) for t in range(T)]  # (m, n) of the CTA's tiles, n fastest
        self.row_blocks = (T + n_tiles - 1) // n_tiles if mode == 3 else 0

    def __repr__(self):
        return (f"S={self.S} K={self.K} T={self.T} mode={self.mode} W={self.W} res={int(self.stage_res)} "
                f"rv={int(self.stage_rv)} cp={int(self.async_bias)}" +
                (f" n_tiles={self.n_tiles}" if self.n_tiles > 1 else ""))


def producer_program(c):
    """the TMA producer thread: per tile and k-iteration `wait_slot(empty_bar(s), ph ^ 1u)` (with stage_res: the
    polling loop that issues a residual whenever `mbar_test_wait(stage_free_bar, r_lt & 1u)` passes), then
    `mbar_arrive_expect_tx(full_bar(s), ...)` and the A / B loads; after the last tile the blocking residual drain"""
    ops = []
    for lt in range(c.T):
        for it in range(c.K):
            j = lt * c.K + it
            if c.mutant == "res_at_top" and it == 0:
                ops.append(("issue_res_now", lt))  # no stage_free probe: the tile's residual goes in at once
            ops += [("wait_slot", j), ("load", j)]
    if c.stage_res and c.mutant != "res_at_top":
        ops.append(("drain_res",))
    return ops


def server_program(c, cta=0):
    """mode 3, lane 31 of the producer warp: one request per tile, then the end marker (s_req_mtile < 0)"""
    ops = []
    for seq in range(1, c.T + 2):
        ops += [("srv_wait", seq, cta), ("srv_ticket", cta), ("srv_reset", cta), ("srv_resp", seq, cta)]
    return ops


def consumer_program(c, lead, storer, cta=0, ring=True):
    """one consumer warp (its lane 0). `lead` is warp 0 (etid 0: the mode-3 mailbox), `storer` issues a TMA store.
    ring=False: the CTA reduced to its mode-3 ticket protocol (the cross-CTA model)"""
    mu = c.mutant
    res, staged = c.stage_res, c.mode != 1 and ring
    ops = [("stage_first",), ("sync", cta)] if ring else [("sync", cta)]  # bias / u of the first tile, epi_sync
    for lt, (m, n) in enumerate(c.tiles):
        # 1. top of the tile: the next tile's bias and u / row-vector row into buffer acc ^ 1 (cp.async, or zeros)
        if ring:
            ops.append(("next_bias", lt))
        # 2. main loop
        for it in range(c.K if ring else 0):
            j = lt * c.K + it
            ops += [("wait_full", j), ("wgmma", j)]
            arrive = [("arrive_empty", j - 1)] if it > 0 else []
            if mu == "early_empty":
                ops += arrive + [("wgmma_wait", 1)]
            else:
                ops += [("wgmma_wait", 1)] + arrive
            if res and it == 0:
                free = [("syncwarp",), ("bulk_wait_read",), ("arrive_stage_free",)]
                if mu == "free_before_read_wait":
                    free = [("syncwarp",), ("arrive_stage_free",), ("bulk_wait_read",)]
                elif mu == "free_without_syncwarp":
                    free = free[1:]
                ops += free
        # 3. drain
        if ring:
            ops += [("wgmma_wait", 0), ("arrive_empty", lt * c.K + c.K - 1)]
        # 4. the previous stores have read the staging tile; epi_sync
        if staged and not (mu == "no_read_wait_unstaged" and not res):
            ops.append(("bulk_wait_read",))
        ops.append(("sync", cta))
        # 5. epilogue, first stage
        if res:
            if mu != "res_full_no_wait":
                ops.append(("wait_res_full", lt ^ 1 if mu == "res_full_parity" else lt))
            ops.append(("epi_res", lt))  # ldmatrix of the residual, stmatrix of the result in place
        elif staged:
            ops.append(("epi_write", lt))
        if ring:
            ops.append(("read_bias", lt))  # sbias, su[acc] (with stage_rv: the row vector)
        if c.mode == 3:
            ops.append(("records", m))
        if ring and mu != "no_cp_wait":
            ops.append(("cp_wait",))
        if c.mode == 3 and lead and lt > 0:
            ops.append(("verdict", lt, cta))  # of tile lt - 1 (request number lt)
        if staged:
            ops += [("fence_async", lt), ("srow_write", lt)]
        # 6. epi_sync
        ops.append(("sync", cta))
        # 7. epilogue, second stage
        if c.mode == 3:
            if lt > 0:
                ops.append(("fold", lt, c.tiles[lt - 1][0], cta))
            if lead:
                ops.append(("post", lt + 1, m, cta))
        if storer:
            ops.append(("store", lt))
        if c.stats:
            ops.append(("stats", lt))
    # 8. mode-3 tail and bulk_wait_all
    if c.mode == 3:
        if mu != "tail_verdict_unsynced":
            ops.append(("sync", cta))  # every warp has read the last tile's verdict before etid 0 overwrites it
        if lead and c.T > 0:
            ops.append(("verdict", c.T, cta))
        ops.append(("sync", cta))
        if c.T > 0:
            ops.append(("fold", c.T, c.tiles[-1][0], cta))
        if lead:
            ops.append(("post", c.T + 1, -1, cta))
    if staged:
        ops.append(("bulk_wait_all",))
    return ops


def splitk_programs(W, mutant=None):
    """the split-K pair's hand-over after the main loop (one work item per CTA). The donor (CTA 1) writes its partial
    tile to the workspace after epi_sync, runs cp_async_wait_all and __threadfence, epi_sync, and warp 0 sets the flag
    after a second __threadfence; the owner (CTA 0) spins on the flag, resets it, and reads the workspace after
    epi_sync"""
    donor = [("sync", 1), ("ws_write",), ("cp_wait",), ("fence_own",), ("sync", 1)]
    donor_lead = donor + [("fence_rel",), ("set_flag",)]
    if mutant == "flag_before_fence":
        donor_lead = donor + [("set_flag",), ("fence_rel",)]
    elif mutant == "flag_before_barrier":
        donor_lead = donor[:4] + [("fence_rel",), ("set_flag",), ("sync", 1)]
    owner = [("bulk_wait_read",), ("sync", 0), ("read_ws",)]
    owner_lead = [("spin_flag",), ("fence_own",), ("reset_flag",)] + owner
    progs = {("own", 1): owner_lead, ("own", 0): owner, ("don", 1): donor_lead, ("don", 0): donor}
    roles = [("own", 1), ("don", 1)] + [("own", 0)] * (W - 1) + [("don", 0)] * (W - 1)
    return progs, roles


# =========================================================================== the interpreter
# shared state, one tuple; fields by index
(F_FULL, F_EMPTY, F_SFREE, F_RFULL, F_STAGE, F_EPI, F_STG, F_BUF, F_SROW, F_MBOX, F_SLAST, F_TICKET, F_RECS, F_FOLDS,
 F_WS, F_FLAG) = range(16)


def _passed(phases, parity):
    return (phases & 1) != parity


def _bump(bar, count):
    """one arrival on an mbarrier (phases, pending) expecting `count` arrivals per phase"""
    c, pnd = bar
    pnd += 1
    return (c + 1, 0) if pnd == count else (c, pnd)


def _tables(progs):
    """per program and pc: the last tile whose read of the bias buffer / the staging tile (epilogue + statistics
    pass) / s_row is complete, and the tile whose staging-tile use is in progress"""
    tab = {}
    for role, ops in progs.items():
        bias, stg_done, stg_in, stats = [], [], [], []
        b = s = st = -1
        cur = -1
        for op in ops + [("end",)]:
            bias.append(b)
            stg_done.append(s)
            stg_in.append(cur)
            stats.append(st)
            if op[0] == "read_bias":
                b = op[1]
            if op[0] in ("epi_res", "epi_write"):
                cur = op[1]
            if op[0] == "stats":
                st = op[1]
        # a tile's staging-tile use ends with its last access (statistics pass, store or epilogue write)
        last = {}
        for k, op in enumerate(ops):
            if op[0] in ("epi_res", "epi_write", "store", "stats"):
                last[op[1]] = k
        for k in range(len(ops) + 1):
            t = stg_in[k]
            if t >= 0 and k > last[t]:
                stg_done[k] = t
        tab[role] = (bias, stg_done, stg_in, stats)
    return tab


def explore(c=None, mutant=None, splitk=None, ctas=None, max_states=5_000_000):
    """all interleavings of one configuration; returns the number of distinct states; raises Violation.
    `c`: a Config (one CTA); `splitk=W`: the split-K pair; `ctas=(G, num_tiles, n_tiles)`: mode 3 across CTAs"""
    if splitk is not None:
        W = splitk
        progs, roles = splitk_programs(W, mutant)
        S, T, W_cta, ncta, n_tiles, rblocks = 1, 0, W, 2, 1, 0
        cfg = None
    elif ctas is not None:
        G, num_tiles, n_tiles = ctas
        progs, roles = {}, []
        for g in range(G):
            tiles = [(t // n_tiles, t % n_tiles) for t in range(g, num_tiles, G)]
            cg = Config(1, 1, len(tiles), 3, W=1, storers=0, n_tiles=n_tiles, mutant=mutant)
            cg.tiles, cg.stats = tiles, False
            progs[("lead", g)] = consumer_program(cg, True, False, cta=g, ring=False)
            progs[("srv", g)] = server_program(cg, g)
            roles += [("lead", g), ("srv", g)]
        S, T, W_cta, ncta, rblocks = 1, 0, 1, G, (num_tiles + n_tiles - 1) // n_tiles
        cfg = None
    else:
        cfg = c
        S, T, W_cta, ncta, n_tiles, rblocks = c.S, c.T, c.W, 1, c.n_tiles, c.row_blocks
        progs = {("prod", 0): producer_program(c)}
        roles = [("prod", 0)]
        for w in range(c.W):
            role = ("lead", 0) if w == 0 else ("store", 0) if w < c.storers else ("plain", 0)
            if role not in progs:
                progs[role] = consumer_program(c, w == 0, w < c.storers)
            roles.append(role)
        if c.mode == 3:
            progs[("srv", 0)] = server_program(c)
            roles.append(("srv", 0))
    tab = _tables(progs)
    mut = cfg.mutant if cfg is not None else mutant
    stats = cfg is not None and cfg.stats
    consumer_kinds = ("lead", "store", "plain", "own", "don")

    # thread: (role, pc, loc); consumer loc = (groups, bulk, cp, lag, joined, rel); producer loc = (r_lt,);
    # server loc = (mt, t)
    def init_loc(role):
        if role[0] == "prod":
            return (0,)
        if role[0] == "srv":
            return (0, -1)
        return ((), (), -1, -1, -1, 0)

    threads = tuple(sorted((r, 0, init_loc(r)) for r in roles))
    shared = [None] * 16
    shared[F_FULL] = (0,) * S
    shared[F_EMPTY] = ((0, 0),) * S
    shared[F_SFREE] = (0, 0)
    shared[F_RFULL] = 0
    shared[F_STAGE] = ((-1, True),) * S
    shared[F_EPI] = ((0, 0),) * ncta
    shared[F_STG] = (-1, True, -1, 0, 0)  # residual tile, landed, result tile, warps written, warps fenced
    shared[F_BUF] = ((-1, 0), (-1, 0))  # (tile, slices landed) of the two bias / u buffers
    shared[F_SROW] = (-1, 0)
    shared[F_MBOX] = ((0, 0, 0, 0),) * ncta  # s_req_seq, s_req_mtile, s_resp_seq, s_resp_last
    shared[F_SLAST] = ((0, 0),) * ncta  # (request number, verdict) of s_last_tile
    shared[F_TICKET] = (0,) * rblocks
    shared[F_RECS] = (0,) * rblocks
    shared[F_FOLDS] = (0,) * rblocks
    shared[F_WS] = (0, 0)  # workspace slices written, slices published by the flag
    shared[F_FLAG] = 0
    init = (tuple(shared), threads)

    def issue_res(sh, ths, r):
        """the residual of local tile r goes into the staging tile (TMA, landing later)"""
        for role, pc, loc in ths:
            if role[0] in consumer_kinds:
                if any(not rd for _, rd in loc[1]):
                    raise Violation(f"staging tile: residual TMA write of tile {r} while a TMA store still reads "
                                    f"tile {[t for t, rd in loc[1] if not rd]}")
                if loc[3] >= 0:
                    raise Violation(f"staging tile: residual TMA write of tile {r} under the statistics pass of "
                                    f"tile {loc[3]} (lanes past lane 0 still read it)")
                _, done, inside, _ = (x[pc] for x in tab[role])
                if inside > done:
                    raise Violation(f"staging tile: residual TMA write of tile {r} while a warp is still in the "
                                    f"epilogue / statistics pass of tile {inside}")
        sh[F_STG] = (r, False, -1, 0, 0)

    def thread_step(st, i):
        """successor states of thread i taking its next op (empty: blocked or done)"""
        shared, ths = st
        role, pc, loc = ths[i]
        ops = progs[role]
        if pc >= len(ops):
            return []
        op = ops[pc]
        k = op[0]
        sh = list(shared)
        out = []

        def moved(pc2=pc + 1, loc2=loc, sh2=None):
            t2 = ths[:i] + ((role, pc2, loc2),) + ths[i + 1:]
            return (tuple(sh if sh2 is None else sh2), tuple(sorted(t2)))

        # ---------------- producer
        if k == "wait_slot":
            j = op[1]
            s, par = j % S, ((j // S) & 1) ^ 1
            (r_lt,) = loc
            if cfg.stage_res and mut != "res_at_top" and r_lt < T and _passed(sh[F_SFREE][0], r_lt & 1):
                sh2 = list(sh)
                issue_res(sh2, ths, r_lt)
                out.append(moved(pc, (r_lt + 1,), sh2))  # poll_res: issue_res(), still waiting for the slot
            if _passed(sh[F_EMPTY][s][0], par):
                out.append(moved())
            return out
        if k == "issue_res_now":
            issue_res(sh, ths, loc[0])
            return [moved(loc2=(loc[0] + 1,))]
        if k == "load":
            j = op[1]
            s = j % S
            for role2, _, loc2 in ths:
                if role2[0] in consumer_kinds:
                    rd = [g for g in loc2[0] if g % S == s]
                    if rd:
                        raise Violation(f"ring stage {s}: TMA load of k-iteration {j} under the unretired wgmma group "
                                        f"of k-iteration {rd[0]}")
            sh[F_STAGE] = sh[F_STAGE][:s] + ((j, False),) + sh[F_STAGE][s + 1:]
            return [moved()]
        if k == "drain_res":
            (r_lt,) = loc
            if r_lt == T:
                return [moved()]
            if _passed(sh[F_SFREE][0], r_lt & 1):
                issue_res(sh, ths, r_lt)
                return [moved(pc, (r_lt + 1,))]
            return []
        # ---------------- ticket server (mode 3)
        if k == "srv_wait":
            seq, g = op[1], op[2]
            req_seq, req_mt, _, _ = sh[F_MBOX][g]
            if req_seq < seq:
                return []
            if req_mt < 0:
                return [moved(len(ops), (req_mt, -1))]  # the epilogue is done
            return [moved(loc2=(req_mt, -1))]
        if k == "srv_ticket":
            mt = loc[0]
            t = sh[F_TICKET][mt]
            sh[F_TICKET] = sh[F_TICKET][:mt] + (t + 1,) + sh[F_TICKET][mt + 1:]
            last = t == n_tiles - 1
            last_reset = t == n_tiles if mut == "ticket_reset_count" else last
            g = op[1]
            rs, rm, ps, _ = sh[F_MBOX][g]
            sh[F_MBOX] = sh[F_MBOX][:g] + ((rs, rm, ps, 1 if last else 0),) + sh[F_MBOX][g + 1:]
            return [moved(loc2=(mt, t if last_reset else -1))]
        if k == "srv_reset":
            mt, t = loc
            if t >= 0:
                sh[F_TICKET] = sh[F_TICKET][:mt] + (0,) + sh[F_TICKET][mt + 1:]
            return [moved(loc2=(mt, -1))]
        if k == "srv_resp":
            seq, g = op[1], op[2]
            rs, rm, _, pl = sh[F_MBOX][g]
            sh[F_MBOX] = sh[F_MBOX][:g] + ((rs, rm, seq, pl),) + sh[F_MBOX][g + 1:]
            return [moved()]

        # ---------------- consumer warps
        groups, bulk, cp, lag, joined, rel = loc
        W = W_cta
        if k == "sync":
            b = op[1]
            gen, pend = sh[F_EPI][b]
            if joined >= 0:
                return [moved(loc2=(groups, bulk, cp, lag, -1, rel))] if gen > joined else []
            pend += 1
            gen2, pend2 = (gen + 1, 0) if pend == W else (gen, pend)
            sh[F_EPI] = sh[F_EPI][:b] + ((gen2, pend2),) + sh[F_EPI][b + 1:]
            # every lane of the warp arrives: its shared-memory reads are complete
            return [moved(pc, (groups, bulk, cp, -1, gen, rel))]
        if k == "syncwarp":
            return [moved(loc2=(groups, bulk, cp, -1, joined, rel))]
        if k == "wait_full":
            j = op[1]
            return [moved()] if _passed(sh[F_FULL][j % S], (j // S) & 1) else []
        if k == "wgmma":
            j = op[1]
            s = j % S
            if sh[F_STAGE][s] != (j, True):
                raise Violation(f"ring stage {s}: the wgmma of k-iteration {j} reads a stage holding "
                                f"{sh[F_STAGE][s]}")
            return [moved(loc2=(groups + (j,), bulk, cp, lag, joined, rel))]
        if k == "wgmma_wait":
            n = op[1]
            return [moved(loc2=(groups[len(groups) - n:] if n else (), bulk, cp, lag, joined, rel))]
        if k == "arrive_empty":
            s = op[1] % S
            sh[F_EMPTY] = sh[F_EMPTY][:s] + (_bump(sh[F_EMPTY][s], W),) + sh[F_EMPTY][s + 1:]
            return [moved()]
        if k == "arrive_stage_free":
            sh[F_SFREE] = _bump(sh[F_SFREE], W)
            return [moved()]
        if k == "bulk_wait_read":
            return [moved()] if all(rd for _, rd in bulk) else []
        if k == "bulk_wait_all":
            return [moved()] if not bulk else []
        if k == "stage_first":
            t, n = sh[F_BUF][0]
            sh[F_BUF] = ((0, n + 1 if t == 0 else 1), sh[F_BUF][1])
            return [moved()]
        if k == "next_bias":
            lt = op[1]
            b = (lt + 1) & 1
            for role2, pc2, _ in ths:
                if role2[0] in consumer_kinds and lt >= 1 and tab[role2][0][pc2] < lt - 1:
                    raise Violation(f"bias/u buffer {b}: tile {lt} writes the next tile's values while a warp has "
                                    f"not read tile {lt - 1}'s")
            t, n = sh[F_BUF][b]
            if lt + 1 < T and cfg.async_bias:  # cp.async: lands later
                if t != lt + 1:
                    sh[F_BUF] = sh[F_BUF][:b] + ((lt + 1, 0),) + sh[F_BUF][b + 1:]
                return [moved(loc2=(groups, bulk, lt + 1, lag, joined, rel))]
            sh[F_BUF] = sh[F_BUF][:b] + ((lt + 1, n + 1 if t == lt + 1 else 1),) + sh[F_BUF][b + 1:]  # plain zeros
            return [moved()]
        if k == "cp_wait":
            return [moved()] if cp < 0 else []
        if k == "read_bias":
            lt = op[1]
            if sh[F_BUF][lt & 1] != (lt, W):
                raise Violation(f"bias/u buffer {lt & 1}: tile {lt} reads it holding {sh[F_BUF][lt & 1]} "
                                f"(tile, slices landed)")
            return [moved()]
        if k == "wait_res_full":
            return [moved()] if _passed(sh[F_RFULL], op[1] & 1) else []
        if k in ("epi_res", "epi_write"):
            lt = op[1]
            rt, landed, ot, oc, fc = sh[F_STG]
            if k == "epi_res" and (rt, landed) != (lt, True):
                raise Violation(f"staging tile: the epilogue of tile {lt} reads the residual of tile {rt} "
                                f"({'landed' if landed else 'not landed'})")
            if k == "epi_write":
                for role2, _, loc2 in ths:
                    if role2[0] in consumer_kinds and any(not rd for _, rd in loc2[1]):
                        raise Violation(f"staging tile: the epilogue of tile {lt} writes it while a TMA store "
                                        f"still reads it")
            sh[F_STG] = (rt, landed, lt, oc + 1 if ot == lt else 1, fc if ot == lt else 0)
            return [moved()]
        if k == "fence_async":
            rt, landed, ot, oc, fc = sh[F_STG]
            if ot == op[1]:
                sh[F_STG] = (rt, landed, ot, oc, fc + 1)
            return [moved()]
        if k == "srow_write":
            lt = op[1]
            for role2, pc2, loc2 in ths:
                if role2[0] in consumer_kinds and stats and lt >= 1 and (tab[role2][3][pc2] < lt - 1 or
                                                                              loc2[3] >= 0):
                    raise Violation(f"s_row: tile {lt} writes it before tile {lt - 1}'s statistics pass has read it")
            t, n = sh[F_SROW]
            sh[F_SROW] = (lt, n + 1 if t == lt else 1)
            return [moved()]
        if k == "store":
            lt = op[1]
            rt, landed, ot, oc, fc = sh[F_STG]
            if (ot, oc, fc) != (lt, W, W):
                raise Violation(f"staging tile: the TMA store of tile {lt} reads it holding the results of tile {ot} "
                                f"from {oc} warps, {fc} of them fenced (residual of tile {rt})")
            return [moved(loc2=(groups, bulk + ((lt, False),), cp, lag, joined, rel))]
        if k == "stats":
            lt = op[1]
            rt, landed, ot, oc, fc = sh[F_STG]
            if (ot, oc) != (lt, W):
                raise Violation(f"staging tile: the statistics pass of tile {lt} reads it holding the results of "
                                f"tile {ot} from {oc} warps (residual of tile {rt})")
            if sh[F_SROW] != (lt, W):
                raise Violation(f"s_row: the statistics pass of tile {lt} reads {sh[F_SROW]}")
            return [moved(loc2=(groups, bulk, cp, lt, joined, rel))]
        if k == "records":
            m = op[1]
            sh[F_RECS] = sh[F_RECS][:m] + (sh[F_RECS][m] + 1,) + sh[F_RECS][m + 1:]
            return [moved()]
        if k == "verdict":
            seq, g = op[1], op[2]
            _, _, ps, pl = sh[F_MBOX][g]
            if ps < seq:
                return []
            if ps != seq:
                raise Violation(f"verdict: request {seq} reads the response to request {ps}")
            sh[F_SLAST] = sh[F_SLAST][:g] + ((seq, pl),) + sh[F_SLAST][g + 1:]
            return [moved()]
        if k == "post":
            seq, m, g = op[1], op[2], op[3]
            rs, _, ps, pl = sh[F_MBOX][g]
            if ps != rs:
                raise Violation(f"verdict: request {seq} overwrites request {rs} before its response")
            sh[F_MBOX] = sh[F_MBOX][:g] + ((seq, m, ps, pl),) + sh[F_MBOX][g + 1:]
            return [moved()]
        if k == "fold":
            seq, m, g = op[1], op[2], op[3]
            sq, last = sh[F_SLAST][g]
            if sq != seq:
                raise Violation(f"verdict: the fold after request {seq} reads the verdict of request {sq}")
            if last:
                if sh[F_RECS][m] != n_tiles * W:
                    raise Violation(f"row block {m}: folded with {sh[F_RECS][m]} of {n_tiles * W} record slices "
                                    f"written")
                sh[F_FOLDS] = sh[F_FOLDS][:m] + (sh[F_FOLDS][m] + 1,) + sh[F_FOLDS][m + 1:]
            return [moved()]
        # split-K
        if k == "ws_write":
            w, p_ = sh[F_WS]
            sh[F_WS] = (w + 1, p_)
            return [moved()]
        if k == "fence_own":
            return [moved()]
        if k == "fence_rel":  # cumulative: every write ordered before it (through the barrier) is published by the flag
            return [moved(loc2=(groups, bulk, cp, lag, joined, sh[F_WS][0]))]
        if k == "set_flag":
            sh[F_FLAG] = 1
            sh[F_WS] = (sh[F_WS][0], rel)
            return [moved()]
        if k == "spin_flag":
            return [moved()] if sh[F_FLAG] == 1 else []
        if k == "reset_flag":
            sh[F_FLAG] = 0
            return [moved()]
        if k == "read_ws":
            if sh[F_WS][1] != W:
                raise Violation(f"split-K workspace: the owner reads it with {sh[F_WS][1]} of {W} donor slices "
                                f"published ({sh[F_WS][0]} written)")
            return [moved()]
        raise AssertionError(f"unknown op {op}")

    def async_events(st):
        shared, ths = st
        out = []
        for s, (j, landed) in enumerate(shared[F_STAGE]):
            if not landed:  # the k-iteration's bytes land: full_bar completes its phase
                sh = list(shared)
                sh[F_STAGE] = shared[F_STAGE][:s] + ((j, True),) + shared[F_STAGE][s + 1:]
                sh[F_FULL] = shared[F_FULL][:s] + (shared[F_FULL][s] + 1,) + shared[F_FULL][s + 1:]
                out.append((tuple(sh), ths))
        rt, landed, ot, oc, fc = shared[F_STG]
        if not landed:  # the residual boxes land: res_full completes its phase
            sh = list(shared)
            sh[F_STG] = (rt, True, ot, oc, fc)
            sh[F_RFULL] = shared[F_RFULL] + 1
            out.append((tuple(sh), ths))
        for i, (role, pc, loc) in enumerate(ths):
            if role[0] not in consumer_kinds or (i > 0 and ths[i - 1] == ths[i]):
                continue
            groups, bulk, cp, lag, joined, rel = loc

            def with_loc(loc2, sh2=shared):
                return (sh2, tuple(sorted(ths[:i] + ((role, pc, loc2),) + ths[i + 1:])))

            if cp >= 0:  # the warp's cp.async lands
                b = cp & 1
                t, n = shared[F_BUF][b]
                buf = shared[F_BUF][:b] + ((cp, n + 1),) + shared[F_BUF][b + 1:]
                sh = shared[:F_BUF] + (buf,) + shared[F_BUF + 1:]
                out.append(with_loc((groups, bulk, -1, lag, joined, rel), sh))
            if bulk:  # the oldest bulk group: its reads complete, then its global writes
                t, rd = bulk[0]
                out.append(with_loc((groups, ((t, True),) + bulk[1:] if not rd else bulk[1:], cp, lag, joined, rel)))
            if lag >= 0:  # the other lanes finish their statistics-pass reads
                out.append(with_loc((groups, bulk, cp, -1, joined, rel)))
        return out

    def check_end(st):
        shared, ths = st
        if not all(pc >= len(progs[role]) for role, pc, _ in ths):
            raise Violation(f"deadlock in state {st}")
        for role, _, loc in ths:
            if role[0] in consumer_kinds and (loc[0] or loc[1] or loc[2] >= 0):
                raise Violation(f"outstanding at exit: a warp ends with wgmma groups {loc[0]}, bulk groups {loc[1]} "
                                f"or a cp.async ({loc[2]}) in flight")
        bars = list(shared[F_EMPTY]) + [shared[F_SFREE]] + list(shared[F_EPI])
        if any(p for _, p in bars):
            raise Violation(f"pending arrivals at the end: {bars}")
        if any(shared[F_TICKET]):
            raise Violation(f"row_ticket: {shared[F_TICKET]} at the end of the launch (a replay would start dirty)")
        if any(f != W_cta for f in shared[F_FOLDS]):
            raise Violation(f"row block: folded {shared[F_FOLDS]} times per block (each warp slice once expected)")
        if shared[F_FLAG]:
            raise Violation("split-K flag: still set at the end of the launch")

    seen = {init}
    todo = deque([init])
    while todo:
        st = todo.popleft()
        succ = async_events(st)
        ths = st[1]
        for i in range(len(ths)):
            if i > 0 and ths[i - 1] == ths[i]:
                continue  # an identical thread: the same successors
            succ += thread_step(st, i)
        if not succ:
            check_end(st)
        for n in succ:
            if n not in seen:
                seen.add(n)
                todo.append(n)
                if len(seen) > max_states:
                    raise RuntimeError("state space larger than expected")
    return len(seen)


def _run(label, **kw):
    t0 = time.perf_counter()
    n = explore(**kw)
    print(f"[gemm protocol] {label}: {n} states, {time.perf_counter() - t0:.2f} s")
    return n


# =========================================================================== configurations
def _configs():
    """W = 2; ring depths 1 / 2 / 3; k-iterations per tile 1, 2 and S + 1 (the ring phase flips inside a tile or at
    its boundary); 1 to 3 tiles per CTA; modes 0 and 3 with and without the staged residual / row vector (without a
    staged row vector the launch has no bias: the top of the tile stores zeros, no cp.async), mode 1 (no staging
    tile) and mode 5. A one-stage ring only serves one k-iteration per tile (see
    test_a_one_stage_ring_needs_one_k_iteration_per_tile). The default run takes the whole matrix for modes 0, 1 and
    5 up to two tiles and, at three, with both staged (or, modes 1 / 5, as they are), and mode 3 (whose ticket server
    multiplies the states) at ring depths 1 and 2 up to two tiles; PP_SLOW_TESTS=1 runs the rest."""
    default, slow = [], []
    for S in (1, 2, 3):
        for K in sorted({1, 2, S + 1}):
            if S == 1 and K > 1:
                continue
            for T in (1, 2, 3):
                for mode in (0, 3):
                    for res, rv in ((False, False), (True, False), (False, True), (True, True)):
                        c = Config(S, K, T, mode, res, rv, bias=False)
                        quick = T < 3 or (res and rv)
                        if mode == 3:
                            quick = S < 3 and T < 3
                        (default if quick else slow).append(c)
                for mode in (1, 5):
                    default.append(Config(S, K, T, mode))
    return default, slow


DEFAULT, SLOW = _configs()


@pytest.mark.parametrize("c", DEFAULT, ids=[repr(c).replace(" ", ",") for c in DEFAULT])
def test_every_interleaving_of_one_cta(c):
    assert _run(repr(c), c=c) > 10


@pytest.mark.skipif(os.environ.get("PP_SLOW_TESTS") != "1", reason="longer runs: set PP_SLOW_TESTS=1")
@pytest.mark.parametrize("c", SLOW, ids=[repr(c).replace(" ", ",") for c in SLOW])
def test_every_interleaving_of_one_cta_rest_of_the_matrix(c):
    assert _run(repr(c), c=c) > 10



@pytest.mark.parametrize("T,n_tiles", [(2, 2), (3, 3), (3, 1)])
def test_mode3_tiles_of_one_row_block_in_one_cta(T, n_tiles):
    """a CTA walking all n-tiles of its row blocks: the verdict of the last one comes a tile late"""
    assert _run(f"mode 3 T={T} n_tiles={n_tiles}", c=Config(1, 1, T, 3, True, True, n_tiles=n_tiles)) > 10


def test_fewer_storing_warps_than_consumer_warps():
    """BLOCK_N = 64 / 128: only warps 0 (and 1) issue a store; the others' stage_free arrivals wait for nothing"""
    assert _run("W=3 storers=1", c=Config(2, 1, 2, 0, True, True, W=3, storers=1)) > 10


@pytest.mark.parametrize("W", [1, 2])
def test_split_k_pair(W):
    assert _run(f"split-K W={W}", splitk=W) > 5


@pytest.mark.parametrize("G,num_tiles,n_tiles", [(2, 2, 1), (2, 4, 2), (2, 3, 3), (2, 6, 3), (3, 3, 3)])
def test_mode3_row_blocks_across_ctas(G, num_tiles, n_tiles):
    """each CTA walks tiles g, g + G, ...; a row block's n-tiles are spread over CTAs and exactly one folds it"""
    assert _run(f"mode 3 across {G} CTAs, {num_tiles} tiles, n_tiles={n_tiles}", ctas=(G, num_tiles, n_tiles)) > 10


# The kernel's ring depths (stages_for: 5 at BLOCK_N 128 / 160, 3 at 256, 8 at 64), one k-iteration per tile, the
# residual and the row vector staged, with as many consumer warps and tiles as this explicit-state search completes
# within 4 M states. Each run's states and seconds on one CPU core (Python 3.12):
#   mode 0, W = 3, 3 tiles: 5 stages 1.81 M / 98 s, 3 stages 1.81 M / 92 s, 8 stages 0.35 M / 15 s
#   mode 0, W = 4: 8 stages, 3 tiles 3.51 M / 191 s; 5 stages, 2 tiles 2.18 M / 95 s
#   mode 3, W = 3: 8 stages, 3 tiles 1.40 M / 74 s; 5 stages, 2 tiles 0.50 M / 21 s
# (about ten minutes in all)
# Past these the search exceeds 4 M states: W = 4 at three tiles with 5 or 3 stages, and mode 3 with W = 3, three
# tiles and 5 stages. The kernel's own eight warps are out of its reach (not run to an end).
KERNEL_RINGS = [  # (W, S, tiles, storing warps, mode)
    (3, 5, 3, 3, 0), (3, 3, 3, 3, 0), (3, 8, 3, 1, 0), (4, 8, 3, 1, 0), (4, 5, 2, 3, 0), (3, 8, 3, 1, 3), (3, 5, 2, 3, 3),
]


@pytest.mark.skipif(os.environ.get("PP_SLOW_TESTS") != "1", reason="longer runs: set PP_SLOW_TESTS=1")
@pytest.mark.parametrize("W,S,T,storers,mode", KERNEL_RINGS, ids=[f"W{w}-S{s}-T{t}-m{m}" for w, s, t, _, m in KERNEL_RINGS])
def test_the_kernels_ring_depths_with_more_warps(W, S, T, storers, mode):
    assert _run(f"kernel rings W={W} S={S} T={T} mode={mode}",
                c=Config(S, 1, T, mode, True, True, W=W, storers=storers), max_states=4_000_000) > 1_000


# =========================================================================== mutants
def test_a_one_stage_ring_needs_one_k_iteration_per_tile():
    """a warp releases stage j - 1 only after it has waited for stage j: one stage deadlocks at two k-iterations
    (why stages_for() never returns fewer than 2)"""
    with pytest.raises(Violation, match="deadlock"):
        explore(Config(1, 2, 1, 0))


@pytest.mark.parametrize("mutant,c,match", [
    ("free_before_read_wait", Config(2, 1, 2, 0, True), "staging tile: residual TMA write .* TMA store still reads"),
    ("free_without_syncwarp", Config(2, 1, 2, 0, True), "staging tile: residual TMA write .* statistics pass"),
    ("res_full_parity", Config(2, 1, 2, 0, True), "staging tile: the epilogue of tile 0 reads the residual"),
    ("res_full_no_wait", Config(2, 1, 1, 0, True), "staging tile: the epilogue of tile 0 reads the residual"),
    ("res_at_top", Config(2, 1, 2, 0, True), "staging tile: .*residual of tile 1"),
    ("early_empty", Config(2, 3, 1, 1), "ring stage 0: TMA load of k-iteration 2 under the unretired"),
    ("no_cp_wait", Config(2, 1, 2, 1), "bias/u buffer 1: tile 1 reads"),
    ("no_read_wait_unstaged", Config(2, 1, 2, 0), "staging tile: the epilogue of tile 1 writes it while a TMA store"),
    ("ticket_reset_count", Config(1, 1, 2, 3, n_tiles=2), "row_ticket"),
    ("tail_verdict_unsynced", Config(1, 1, 2, 3), "verdict: the fold after request 1 reads the verdict of request 2"),
], ids=lambda x: x if isinstance(x, str) and " " not in x else "")
def test_each_mutant_is_visible_to_the_model(mutant, c, match):
    c.mutant = mutant
    with pytest.raises(Violation, match=match):
        explore(c)


@pytest.mark.parametrize("mutant", ["flag_before_fence", "flag_before_barrier"])
def test_an_early_split_k_flag_is_visible_to_the_model(mutant):
    with pytest.raises(Violation, match="split-K workspace"):
        explore(splitk=2, mutant=mutant)


def test_a_wrong_ticket_reset_is_visible_across_ctas():
    with pytest.raises(Violation, match="row_ticket"):
        explore(ctas=(2, 4, 2), mutant="ticket_reset_count")


# =========================================================================== the source
def _read_src():
    with open(SRC) as f:
        return f.read()


def _in_order(text, lines, what):
    pos, at = [], 0
    for x in lines:
        assert x in text[at:], f"gemm_conv.cu: `{x}` missing or out of order in {what}: update the protocol model"
        at = text.index(x, at) + len(x)
        pos.append(at)
    return pos


def check_source(src):
    """every wait, arrival, parity and barrier the programs restate, verbatim in `src` and in their order"""
    start = src.index("gemm_conv_kernel(const __grid_constant__ GemmKParams p) {")
    k = src[start:src.index("// host side", start)]
    for line in [
        "static constexpr int GEMM_EPI_WARPS = 8;                     // two consumer warpgroups",
        "mbar_init(full_bar(s), 1);",
        "mbar_init(empty_bar(s), GEMM_EPI_WARPS);  // one arrival per consumer warp",
        "mbar_init(stage_free_bar, GEMM_EPI_WARPS);",
        "mbar_init(res_full_bar, 1);",
        "static_assert(stages_for(160) == 5 && stages_for(128) == 5 && stages_for(256) == 3 && stages_for(64) == 8,",
        'auto epi_sync = [] { asm volatile("bar.sync 1, %0;" ::"n"(GEMM_EPI_WARPS * 32) : "memory"); };',
        "const bool stage_res = kRes && p.res1 != nullptr && !(kSplitK && khalf);",
    ]:
        assert line in src, f"gemm_conv.cu no longer contains `{line}`: update the protocol model"
    assert GEMM_EPI_WARPS == int(re.search(r"GEMM_EPI_WARPS = (\d+);", src).group(1))

    # ---- producer: the polling wait, the loads, the drain
    prod = k[k.index("// ===================== TMA producer"):k.index("// ===================== consumer warpgroups")]
    _in_order(prod, ["mbar_arrive_expect_tx(res_full_bar, bytes);", "tma_load_2d(s_out_addr + sub * 16384, tm, res_full_bar",
                     "++r_lt;"], "issue_res")
    _in_order(prod, ["while (r_tile < num_tiles && mbar_test_wait(stage_free_bar, r_lt & 1u)) issue_res();"],
              "poll_res")
    _in_order(prod, ["if (!stage_res) {", "mbar_wait(bar, parity);", "poll_res();",
                     "while (!mbar_test_wait(bar, parity)) {", "poll_res();"], "wait_slot")
    _in_order(prod, ["int s = 0;", "uint32_t ph = 0;", "wait_slot(empty_bar(s), ph ^ 1u);", "#else",
                     "mbar_arrive_expect_tx(full_bar(s), p.a_bytes + B_STAGE_BYTES);",
                     "tma_load_2d(dstB, &p.tmB, full_bar(s), it * BLOCK_K, n_tile * BLOCK_N);",
                     "if (++s == STAGES) { s = 0; ph ^= 1u; }",
                     "if (stage_res) {", "while (r_tile < num_tiles) {", "mbar_wait(stage_free_bar, r_lt & 1u);",
                     "issue_res();"], "the producer loop and the residual drain")
    # ---- ticket server
    _in_order(prod, ["while (s_req_seq < seq) {", "const int mt = s_req_mtile;", "if (mt < 0) break;",
                     "__threadfence();", "const int t = atomicAdd(p.row_ticket + mt, 1);",
                     "if (t == n_tiles - 1) p.row_ticket[mt] = 0;", "s_resp_last = (t == n_tiles - 1) ? 1 : 0;",
                     "s_resp_seq = seq;"], "the ticket server")

    cons = k[k.index("// ===================== consumer warpgroups"):]
    # ---- main loop: full wait, wgmma, wait<1>, empty arrival, then the stage_free arrival in the first iteration
    ml = _in_order(cons, ["mbar_wait(full_bar(ks), kph);", "wgmma_commit();", "wgmma_wait<1>();",
                          "if (it > k_begin && lane_id() == 0) mbar_arrive(empty_bar(prev));",
                          "if (stage_res && it == k_begin) {", "__syncwarp();", "if (lane_id() == 0) {",
                          "bulk_wait_read_all();", "mbar_arrive(stage_free_bar);",
                          "if (++ks == STAGES) { ks = 0; kph ^= 1u; }",
                          "wgmma_wait<0>();", "if (lane_id() == 0) mbar_arrive(empty_bar(prev));"], "the main loop")
    # split-K owner spin, then the tile-end read wait and epi_sync
    _in_order(cons[ml[-1]:], ["while (*fl == 0) {", "__threadfence();", "*fl = 0;  // ready for the next launch",
                              "if ((etid & 31) == 0) bulk_wait_read_all();", "epi_sync();", "if (khalf) {",
                              "ws[i * (GEMM_EPI_WARPS * 32)] = make_float4(", "} else {",
                              "const float4 pp = __ldcg(ws + i * (GEMM_EPI_WARPS * 32));"], "the split-K hand-over")
    # top of the tile: the next tile's bias / u / row vector into buffer acc ^ 1
    _in_order(cons, ["const uint32_t acc = lt & 1u;", "const float* sbias = sbias_all + acc * BLOCK_N;",
                     "const float* su = su_all + acc * BLOCK_N;",
                     "float* db = sbias_all + (acc ^ 1u) * BLOCK_N + etid;",
                     "if (next_tile < num_tiles && p.bias && nn < p.N) cp_async_f32(db, p.bias + nn);",
                     "else *db = 0.f;", "else if (next_tile < num_tiles && stage_rv && nn < p.N) cp_async_f32(du, rv_row(tw.m) + nn);",
                     "else *du = 0.f;"], "the top of the tile")
    # epilogue, first stage: residual wait before the first ldmatrix, then the reads of sbias / su and the stmatrix
    lean = cons[cons.index("mainloop(facc, m_tile, n_tile, [&] {"):]
    _in_order(lean, ["if (khalf) {", "cp_async_wait_all();", "__threadfence();", "epi_sync();", "if (etid == 0) {",
                     "__threadfence();", "*(volatile int32_t*)(p.splitk_flags + (int64_t)m_tile * n_tiles + n_tile) = 1;",
                     "continue;"], "the split-K donor")
    _in_order(lean, ["if (stage_res) mbar_wait(res_full_bar, lt & 1u);", "if (stage_res) ldmatrix_x4(st_addr(k), r1q);",
                     "const float2 b = *reinterpret_cast<const float2*>(sbias + c);",
                     ": stage_rv ? *reinterpret_cast<const float2*>(su + c) : tv[k][g][h];",
                     "p.row_stats[(int64_t)(n_tile * 2 + hf) * p.row_stats_ld + row[h]] =",
                     "stmatrix_x4(st_addr(k), pack_bf16x2("], "the epilogue's first stage")
    assert lean.index("if (stage_res) mbar_wait(res_full_bar, lt & 1u);") < lean.index("ldmatrix_x4(st_addr(k)")
    # tile end: cp.async wait, the verdict, the proxy fence and s_row, epi_sync; then the request, the store, the fold,
    # the statistics pass
    end = lean[lean.index("// generic (fp32 / transposed / ragged N)"):]
    _in_order(end, ["cp_async_wait_all();",
                    "if (etid == 0 && lt > 0) s_last_tile = ticket_verdict((int)lt);  // of tile lt - 1 (request number lt)",
                    "fence_proxy_async_smem();  // the staging stores (generic proxy) -> the TMA unit (async proxy)",
                    "s_row[r0] = valid[0] ? (long long)row[0] : -1ll;", "epi_sync();",
                    "fold_prev = lt > 0 && s_last_tile != 0 && prev_valid;",
                    "s_req_mtile = m_tile;", "s_req_seq = (int)lt + 1;",
                    "if ((etid & 31) == 0 && (etid >> 5) * 64 < (MODE == 5 ? BLOCK_N : OUT_COLS)) {",
                    "tma_store_2d(tm, s_out_addr + sub * 16384, col, m_tile * BLOCK_M);", "bulk_commit_group();",
                    "if (fold_prev) fold_row_records(frc, prev_row);",
                    "if constexpr (MODE == 0 || MODE == 3 || MODE == 4) {",
                    "const uint4 q = *reinterpret_cast<const uint4*>(s_out + stage_off(rb, piece * 8));",
                    "if (s_row[rr] >= 0) {",
                    # mode-3 tail and the final bulk wait
                    "epi_sync();", "if (etid == 0 && lt > 0) s_last_tile = ticket_verdict((int)lt);", "epi_sync();",
                    "if (lt > 0 && s_last_tile != 0 && prev_valid) {", "s_req_mtile = -1;", "s_req_seq = (int)lt + 1;",
                    "if ((etid & 31) == 0) bulk_wait_all();"], "the tile end and the mode-3 tail")
    verdict = cons[cons.index("auto ticket_verdict = [&](int seq) -> int {"):]
    _in_order(verdict, ["while (s_resp_seq < seq) {", "return s_resp_last;"], "ticket_verdict")
    # the first tile's bias is staged before an epi_sync, outside the tile loop
    _in_order(cons, ["sbias_all[etid] = b0;", "epi_sync();", "for (int tile = walk_first; tile < num_tiles;"],
              "the first tile's bias")


def test_model_matches_the_source():
    check_source(_read_src())


REORDERED = [  # (the source's lines, swapped): each must fail the check
    ("bulk_wait_read_all();\n                        mbar_arrive(stage_free_bar);",
     "mbar_arrive(stage_free_bar);\n                        bulk_wait_read_all();"),
    ("wgmma_wait<1>();\n                if (it > k_begin && lane_id() == 0) mbar_arrive(empty_bar(prev));",
     "if (it > k_begin && lane_id() == 0) mbar_arrive(empty_bar(prev));\n                wgmma_wait<1>();"),
    ("cp_async_wait_all();\n            if constexpr (MODE == 3) {",
     "if constexpr (MODE == 3) {"),
    ("if (stage_res) mbar_wait(res_full_bar, lt & 1u);", "if (stage_res) mbar_wait(res_full_bar, (lt + 1) & 1u);"),
    ("__syncwarp();\n                    if (lane_id() == 0) {", "if (lane_id() == 0) {"),
    ("if (t == n_tiles - 1) p.row_ticket[mt] = 0;", "if (t == n_tiles) p.row_ticket[mt] = 0;"),
    ("__threadfence();\n                            *(volatile int32_t*)(p.splitk_flags",
     "*(volatile int32_t*)(p.splitk_flags"),
    ("mbar_init(stage_free_bar, GEMM_EPI_WARPS);", "mbar_init(stage_free_bar, 4);"),
]


@pytest.mark.parametrize("old,new", REORDERED, ids=range(len(REORDERED)))
def test_the_source_check_sees_a_removed_or_reordered_line(old, new):
    src = _read_src()
    assert src.count(old) == 1, old
    with pytest.raises(AssertionError, match="gemm_conv.cu"):
        check_source(src.replace(old, new))
