"""The graph phases at their edges: add_alignment, the per-root sort, the subgraph of a partial-span read and the heaviest
bundle.  Window sets in the style of fill_cases.py and tb_cases.py, each named for what it must reach.

racon's offset rule (window.cpp:87-95) counts a layer as spanning the window only if begin < offset and
end > L - offset, offset = (uint32)(0.01 * L).  Below 200 bases offset is 0 or 1, so a read from 0 to L - 1 is a
partial-span layer there: in the cliques, ties, branch and lengths windows (31 to 150 bases) every read is aligned to
a subgraph that is the whole graph, and their sub_begin0 / sub_end_last counts are those reads, not partial layers
proper.  roots, subgraph, limits_indegree, weights and real combine the graph phases with whole-graph alignment.

The CPU suite runs every case through the emulation, which checks the sort, the subgraph and the consensus scores
against their serial twins and counts the paths taken (tests/test_graph_reach.py); in full band the per-read graph,
subgraph and consensus digests must also equal spoa's.  The GPU suite compares the digest build's digests, statuses and
outputs with the emulation's (tests/test_gpu_graph.py).
"""
from __future__ import annotations

import numpy as np

import fill_cases as fc
from fill_cases import ACGT, WindowBatch, _window, run, synth_windows

#: letters of one column, in the order the clique case adds them (the backbone holds the first)
COLUMN = b"ACGTNRYKM"


def clique_windows(k_max: int = 8) -> WindowBatch:
    """Per k in 2..k_max: a column of k distinct letters (ACGT, N, IUPAC) in the middle of a 100-base window, every
    other column plain; each letter carried by two reads so that the clique is also matched, not only joined."""
    rng = np.random.default_rng(31)
    wins = []
    for k in range(2, k_max + 1):
        bb = bytearray(rng.choice(ACGT, 100).tobytes())
        bb[50] = COLUMN[0]
        reads = []
        for j in range(1, k):
            r = bytearray(bb)
            r[50] = COLUMN[j]
            reads += [bytes(r), bytes(r)]
        wins.append(_window([bytes(bb)] + reads, [None] * (len(reads) + 1)))
    return WindowBatch.from_lists(wins)


def tie_windows() -> WindowBatch:
    """Constant weights, symmetric variants split half and half: a SNP every 3 to 9 bases, carried by exactly half the
    sequences (the backbone among them), so that the node after each SNP has two in-edges of equal weight from
    predecessors of equal score.  SNPs fall on both sides of the 32-rank block edges."""
    rng = np.random.default_rng(32)
    wins = []
    for L, depth, step in ((60, 8, 7), (100, 8, 5), (150, 10, 6), (97, 6, 9), (130, 8, 4), (120, 6, 3)):
        bb = bytearray(rng.choice(ACGT, L).tobytes())
        alt = bytearray(bb)
        for p in range(3, L - 3, step):
            alt[p] = int(rng.choice([c for c in ACGT if c != bb[p]]))
        seqs = [bytes(bb)] + [bytes(alt) if i % 2 == 0 else bytes(bb) for i in range(depth - 1)]
        wins.append(_window(seqs, [None] * depth))
    return WindowBatch.from_lists(wins)


def branch_windows() -> WindowBatch:
    """Backbones of weight 0 (racon's '!' dummy quality of a FASTA target) and reads of weight 1 that stop k bases before
    the backbone's end: past the reads the scores stay flat, the heaviest node is not a sink and branch completion runs
    once per remaining node (k = 0: none)."""
    rng = np.random.default_rng(33)
    wins = []
    for k in (0, 1, 2, 5):
        bb = rng.choice(ACGT, 120).tobytes()
        reads = [bb[:120 - k]] * 6
        wins.append(_window([bb] + reads, [np.zeros(120, dtype=np.int8)] + [None] * 6))
    return WindowBatch.from_lists(wins)


def root_windows() -> WindowBatch:
    """Long insertions (40 bases, and 70 Ns) and deletions, and reads with a substitution every 6 bases: one read adds runs of
    more than 32 and 64 new nodes and dirties more than 32 roots of the per-root sort."""
    rng = np.random.default_rng(34)
    wins = []
    for w in range(3):
        bb = rng.choice(ACGT, 300).tobytes()
        reads = []
        for i in range(6):
            ins = rng.choice(ACGT, 40).tobytes() if i % 2 else b"N" * 70  # N matches nothing: 70 new nodes
            reads.append(bb[:100 + 10 * w] + ins + bb[100 + 10 * w:])
            reads.append(bb[:150] + bb[150 + 30 + 5 * i:])
            sub = bytearray(bb)
            for p in range(2 + i, 300, 6):
                sub[p] = int(rng.choice([c for c in ACGT if c != sub[p]]))
            reads.append(bytes(sub))
        wins.append(_window([bb] + reads, [None] * (len(reads) + 1)))
    return WindowBatch.from_lists(wins)


def subgraph_windows() -> WindowBatch:
    """Partial-span layers that begin at backbone node 0 or end at the last backbone node, over graphs whose columns hold
    cliques of up to 8 letters every 5 bases (some of them cut by an edge of the subgraph sweep's 32-rank chunks)."""
    rng = np.random.default_rng(35)
    wins = []
    for w in range(4):
        L = 200 + 40 * w
        bb = bytearray(rng.choice(ACGT, L).tobytes())
        win = [(bytes(bb), None, 0, 0)]
        for j in range(1, 8):
            r = bytearray(bb)
            for p in range(3 + w, L - 3, 5):
                r[p] = COLUMN[(COLUMN.index(bb[p]) + j) % 8] if bb[p] in COLUMN[:8] else bb[p]
            win.append((bytes(r), None, 0, L - 1))
        for i in range(6):
            a = int(rng.integers(L // 4, L // 2))
            if i % 2:
                win.append((bytes(bb[:a]), None, 0, a))              # begins at node 0
            else:
                win.append((bytes(bb[a:]), None, a, L - 1))          # ends at the last node
        wins.append(win)
    return WindowBatch.from_lists(wins)


def big_subgraph_windows() -> WindowBatch:
    """Graphs of more than sroot_cap (about 3.4 k) nodes with partial-span layers: mark_subgraph falls back to
    mark_subgraph_serial."""
    wins = []
    for w in range(2):
        b = synth_windows(1, 1400, 26, 0.3, seed=360 + w)
        seqs, wts, _, _ = b.window(0)
        L = len(seqs[0])
        win = [(seqs[0], wts[0], 0, 0)] + [(s, None, 0, L - 1) for s in seqs[1:20]]
        for s in seqs[20:]:
            win.append((s[300:1000], None, 300, 1000))
        wins.append(win)
    return WindowBatch.from_lists(wins)


#: max_sequence_size of the node-count case: b200poa_config_default gives 3 x 64 = 192 nodes in full band
LIMIT_MSZ = 64


def node_limit_windows() -> WindowBatch:
    """A 64-base backbone and reads that are all N or all R: every such read adds one aligned node per base.  Backbone +
    N + R is exactly 192 = max_nodes nodes; one more read with a single Y makes it 193."""
    rng = np.random.default_rng(37)
    bb = rng.choice(ACGT, LIMIT_MSZ).tobytes()
    y = bytearray(bb)
    y[30] = ord("Y")
    at = [bb, b"N" * LIMIT_MSZ, b"R" * LIMIT_MSZ, b"N" * LIMIT_MSZ]
    over = at + [bytes(y)]
    return WindowBatch.from_lists([_window(at, [None] * 4), _window(over, [None] * 5)])


#: backbone position whose node collects the in-edges of the in-degree case
HUB = 300
#: letters inserted in front of the hub, one per read: every byte but the hub's (N), its predecessor's (R) and '-'
HUB_LETTERS = bytes(c for c in range(1, 256) if c not in b"RN-")


def indegree_windows() -> WindowBatch:
    """A hub node (N, after an R) that collects exactly 255 and exactly 256 in-edges, then one plain read whose row program
    must hold the hub's in-degree: 255 fits the row record, 256 stops the window with ST_EDGE_COUNT_EXCEEDED.

    Each in-edge has a source of its own.  252 reads carry one inserted letter in front of the hub, each a letter no
    other read has: aligning it to an earlier read's inserted node would be a mismatch (-5), worse than inserting it
    (-4), so every such read adds a new node and its edge into the hub.  Two or three reads lack the last 1, 2 or 3
    backbone bases before the hub (distinct bases, so the deletion cannot slide) and add an edge from the node before
    the gap.  Deletions alone do not get far: later reads reuse an earlier skip edge by placing their gap elsewhere."""
    rng = np.random.default_rng(38)
    wins = []
    for n_del in (2, 3):
        bb = bytearray(rng.choice(ACGT, 420).tobytes())
        bb[HUB - 4:HUB - 1] = b"ACG"
        bb[HUB - 1] = ord("R")
        bb[HUB] = ord("N")
        bb = bytes(bb)
        reads = [bb[:HUB - k] + bb[HUB:] for k in range(1, n_del + 1)]
        reads += [bb[:HUB] + bytes([c]) + bb[HUB:] for c in HUB_LETTERS]
        # racon sorts the layers by begin (not stably): the plain read begins at 3, still a full-span layer of a
        # 420-base window (3 < 0.01 * 420), so that it is processed last
        spans = [(0, 0)] + [(0, len(bb) - 1)] * len(reads) + [(3, len(bb) - 1)]
        wins.append(_window([bb] + reads + [bb], [None] * (len(reads) + 2), spans))
    return WindowBatch.from_lists(wins)


#: the hub's in-degree in each window of indegree_windows (the largest in-degree of its final graph)
HUB_INDEGREE = [255, 256]


def length_windows() -> WindowBatch:
    """Consensus lengths 31, 32, 33 and 64 (reads equal to the backbone); and a window of 9 sequences whose 8 reads are
    one base each: such a read bumps no coverage, so no consensus base reaches the trim threshold of (9 - 1) / 2."""
    rng = np.random.default_rng(39)
    wins = []
    for L in (31, 32, 33, 64):
        bb = rng.choice(ACGT, L).tobytes()
        wins.append(_window([bb] * 5, [None] * 5))
    bb = rng.choice(ACGT, 80).tobytes()
    wins.append(_window([bb] + [rng.choice(ACGT, 1).tobytes() for _ in range(8)], [None] * 9))
    return WindowBatch.from_lists(wins)


def weight_windows() -> WindowBatch:
    """FASTQ extremes: per-base weights of 0 ('!') and 93 ('~'), mixed and whole reads of each."""
    rng = np.random.default_rng(40)
    b = synth_windows(4, 200, 12, 0.12, seed=400)
    wins = []
    for w in range(b.n_windows):
        seqs, _, _, _ = b.window(w)
        wts = []
        for i, s in enumerate(seqs):
            n = len(s)
            wts.append({0: np.full(n, 93, dtype=np.int8), 1: np.zeros(n, dtype=np.int8)}.get(
                i % 4, rng.choice(np.array([0, 93], dtype=np.int8), n)))
        wins.append(_window(list(seqs), wts))
    return WindowBatch.from_lists(wins)


def real_runs():
    from common import cudapoa_fixture, lambda_fixture
    out = []
    for case in ("fastq_500", "fasta_500", "fastq_1000"):
        out.append(run(f"real_lambda_{case}", lambda_fixture(case)[0], msz=1279 if case.endswith("1000") else 1023))
    cb, _, _ = cudapoa_fixture()
    out.append(run("real_cudapoa", cb, msz=2047, depth=256))
    return out


def cases():
    """name -> list of runs (fill_cases.run)."""
    out = {}
    out["cliques"] = [run("cliques_full", clique_windows()), run("cliques_static", clique_windows(), mode="static")]
    out["ties"] = [run("ties_full", tie_windows()), run("ties_static", tie_windows(), mode="static", band=128)]
    out["branch"] = [run("branch_full", branch_windows())]
    out["roots"] = [run("roots_full", root_windows()), run("roots_adaptive", root_windows(), mode="adaptive", band=64)]
    out["subgraph"] = [run("subgraph_full", subgraph_windows()),
                       run("subgraph_big", big_subgraph_windows(), msz=2047)]
    out["limits"] = [run("limits_aligned", WindowBatch.from_lists([list(zip(*clique_windows(9).window(7)))])),
                     run("limits_nodes", node_limit_windows(), msz=LIMIT_MSZ),
                     run("limits_indegree", indegree_windows(), depth=257)]
    out["lengths"] = [run("lengths_full", length_windows())]
    out["weights"] = [run("weights_full", weight_windows()), run("weights_static", weight_windows(), mode="static")]
    out["real"] = real_runs()
    return out


#: what each limits run must report per window (status codes of poa_core.cuh Status)
LIMIT_STATUS = {"limits_aligned": [11], "limits_nodes": [0, 4], "limits_indegree": [0, 5]}


def reach_failures(case: str, r, out) -> list:
    """The unmet promises of one run, from the emulation's graph report."""
    rep, st = out["graph_reach"], out["status"]
    tot = {k: int(v.sum()) for k, v in rep.items()}
    b = r["batch"]
    need = []

    def want(*fields):
        for f in fields:
            if tot[f] == 0:
                need.append(f"{r['name']}: {f} never reached")

    name = r["name"]
    if name in LIMIT_STATUS:
        if st.tolist() != LIMIT_STATUS[name]:
            need.append(f"{name}: statuses {st.tolist()} != {LIMIT_STATUS[name]}")
    elif (st != 0).any():
        need.append(f"{name}: statuses {st.tolist()}")
    want("topsort_twins")
    if not name.startswith("limits"):
        want("cons_twins")
    if case == "cliques":
        want(*[f"join{k}" for k in range(1, 8)], "const_weights")
    elif case == "ties":
        want("tie_in_block", "tie_pre_block", "tie_equal_pred", "block_max_tie")
    elif case == "branch":
        rounds = out["graph"]["cons_rounds"]
        if not ((rounds == 0).any() and (rounds == 1).any() and (rounds >= 2).any()):
            need.append(f"{name}: branch-completion rounds {rounds.tolist()}: not 0, 1 and 2 or more")
    elif case == "roots":
        want("new_nodes32", "new_nodes64", "run_cross32", "dirty_over32", "edge_same_root", "edge_cross_root",
             "edge_bumped", "du_all")
    elif case == "subgraph":
        if name == "subgraph_big":
            want("sub_serial")
        else:
            want("sub_begin0", "sub_end_last", "sub_twins", "sweep_iter2", "straddle", "straddle8")
    elif case == "limits" and name == "limits_indegree":
        want("walk_over32", "edge_created")
    elif case == "lengths":
        want("read_len1")
        L = [len(c) for c in out["cons"]]
        if sorted({x % 32 for x in L[:4]}) != [0, 1, 31]:
            need.append(f"{name}: consensus lengths {L}")
        trim = int(out["trim"][4])
        if (trim & 0xFFFF) <= (trim >> 16):
            need.append(f"{name}: a base of window 4 passes the trim threshold")
    elif case == "weights":
        want("weight0", "base_weights")
    elif case == "real":
        want("clique_mate", "new_nodes32", "edge_bumped")
    if tot["twin_mismatches"]:
        need.append(f"{name}: {tot['twin_mismatches']} twin mismatches")
    return need


def mismatch_report(r, out) -> list:
    """The first graph twin mismatch of every window, named by window and read."""
    kinds = {0: "sort", 1: "subgraph", 2: "consensus scores"}
    bad = []
    for w, m in enumerate(out["graph_mismatch"]):
        if m[0] >= 0:
            where = f"read {m[1]}" if m[0] != 2 else "consensus"
            bad.append(f"{r['name']}: window {w} {where}: {kinds[int(m[0])]} differ from the serial twin at "
                       f"{m[2]}: twin {m[3]}, engine {m[4]}")
    return bad


def oracle_graph(oracle, r) -> dict:
    from racon_gpu_b200 import api
    m, x, g = r["scoring"]
    return oracle.graph_digests(r["batch"], api.processing_order(r["batch"]), m, x, g)
