"""Ping-pong tile engine on the CPU: a restatement of the tile choice for every conv launch of the encoder (geometry()
follows conv_geometry in csrc/encoder.cu decision by decision, in the same order), and a model of the pipeline protocol
of a ping-pong launch (tile_gemm.cuh, gemm_consumer_pingpong).

The protocol model runs the TMA producer, the two consumer warpgroups, the shared-memory ring (full / empty mbarriers
with phase parity) and the order barrier (turn_bar) as interleaved agents under a seeded random schedule.  TMA loads
and wgmma groups complete asynchronously, in any order the schedule picks (wgmma groups of one warpgroup in order).  A
run reports what went wrong: a deadlock, a slot read out of the producer's order, a slot read before it holds its
k-block, a slot overwritten while a wgmma group still reads it, or a slot not filled, read and released exactly once."""
import dataclasses
import random
from typing import Dict, List, Optional

# ------------------------------------------------------------------------------------------- conv_geometry, restated
NUM_SMS = 132
SMEM_LIMIT = 227 * 1024
TILE_A = 128 * 64 * 2
HALO_PIECE = 23 * 1024
MODES = {"fp32": 3, "bf16x2": 2, "bf16": 1, "fp16x2": 2, "fp16": 1}     # operand pieces per mode
PINGPONG_MAX_KB = 32                                                     # k-blocks per tile (at block_n 64)


def _ceil(a, b):
    return -(-a // b)


def pick_block_n(cout):
    if cout % 128 == 0:
        return 128
    if cout % 64 == 0:
        return 64
    return 80 if cout <= 80 else 96


def pick_tile(Wo, Ho):
    w = 1
    while w < Wo and w < 128:
        w <<= 1
    h = 1
    while h < Ho and w * h < 128:
        h <<= 1
    return w, h, 128 // (w * h)


def fixed_smem(block_n, frag_epi):
    acc = 0 if frag_epi else 128 * _ceil(block_n, 32) * 32 * 4
    return 8 * 4096 + acc + 1024 + 512


def max_stages(P, block_n, frag_epi):
    return min(8, (SMEM_LIMIT - fixed_smem(block_n, frag_epi)) // (P * TILE_A + P * block_n * 64 * 2))


def halo_b_stages(P, block_n, frag_epi):
    return min(8, (SMEM_LIMIT - fixed_smem(block_n, frag_epi) - 2 * P * HALO_PIECE) // (P * block_n * 64 * 2))


@dataclasses.dataclass
class Launch:
    layer: str
    N: int
    H: int                 # input map
    W: int
    C: int
    cout: int
    R: int = 1
    S: int = 1
    stride: int = 1
    pad: int = 0
    res_mode: int = 0      # 1 residual, 2 gate, 4 second 1x1 source of res_C channels
    res_C: int = 0
    frag_epi: bool = True
    stem: bool = False
    sparse: bool = False
    parity: int = 0
    identity: bool = False


def network(B: int, td_parity: bool = False, heat_sparse: bool = True) -> List[Launch]:
    """The conv launches of build_graph, in plan order."""
    L = []
    L.append(Launch("stem", B, 128, 132, 16, 64, R=4, stem=True))
    H, C = 64, 64

    def stage(si, H, C):
        mid, out = (64, 256) if si == 0 else (128, 512) if si == 1 else (256, 1024) if si == 2 else (512, 2048)
        for ui in range({0: 3, 1: 4, 2: 6, 3: 3}[si]):
            p = f"s{si + 1}u{ui + 1}"
            st = 2 if ui == 0 and si != 0 else 1
            L.append(Launch(p + "c1", B, H, H, C, mid, stride=st))
            Ho = (H - 1) // st + 1
            L.append(Launch(p + "c2", B, Ho, Ho, mid, mid, R=3, S=3, pad=1))
            if ui == 0:
                L.append(Launch(p + "c3", B, Ho, Ho, mid, out, res_mode=4, res_C=C))
            else:
                L.append(Launch(p + "c3", B, Ho, Ho, mid, out, res_mode=1, identity=True))
            H, C = Ho, out
        return H, C

    for si in range(3):
        H, C = stage(si, H, C)
    L.append(Launch("lat4", B, 32, 32, 512, 256))
    L.append(Launch("lat5", B, 16, 16, 1024, 256))
    L.append(Launch("lat6", B, 16, 16, 1024, 256, R=3, S=3, stride=2, pad=1))
    L.append(Launch("lat7", B, 8, 8, 256, 256, R=3, S=3, stride=2, pad=1))
    for li in range(2):
        p = f"b{li}_"
        for lvl, hs in (("p6td", 8), ("p5td", 16), ("p4td", 32), ("p3td", 64)):
            if not td_parity or hs < 32:
                L.append(Launch(p + lvl + "_u", B, hs // 2, hs // 2, 256, 256))
                L.append(Launch(p + lvl, B, hs, hs, 256, 256, res_mode=1, identity=True))
            else:
                L.append(Launch(p + lvl + "_u", B, hs // 2, hs // 2, 256, 256))
                for ab in range(4):
                    L.append(Launch(p + lvl, B, hs, hs, 256, 256, stride=2, res_mode=1, identity=True, parity=1 + ab))
        for lvl, hs in (("p4out", 32), ("p5out", 16), ("p6out", 8), ("p7out", 4)):
            L.append(Launch(p + lvl, B, hs, hs, 256, 256))
    heat = dict(R=3, S=3, pad=1, frag_epi=False)
    L.append(Launch("heat", B, 64, 64, 256, 68, **heat))
    if heat_sparse:
        L.append(Launch("heat", B, 64, 64, 256, 68, sparse=True, **heat))
    L.append(Launch("fusion", B, 16, 16, 1408, 1024, res_mode=2))
    stage(3, 16, 1024)
    L.append(Launch("mlp1", 1, 1, B, 2048, 1536))
    L.append(Launch("mlp2", 1, 1, B, 1536, 549, frag_epi=False))
    return L


def geometry(ln: Launch, P: int, use_halo: bool = True) -> Dict[str, int]:
    """The GemmGeom fields (and launch grid) conv_geometry derives for one launch, as describe_plan names them; in the
    order of conv_geometry, so that the two read side by side."""
    bn_w = pick_block_n(ln.cout)
    cout_pad = _ceil(ln.cout, bn_w) * bn_w
    has_b64 = bn_w == 128
    if ln.stem:
        Ho, Wo = ln.H, ln.W - 4
    elif ln.parity:
        Ho, Wo = ln.H // 2, ln.W // 2
    else:
        Ho = (ln.H + 2 * ln.pad - ln.R) // ln.stride + 1
        Wo = (ln.W + 2 * ln.pad - ln.S) // ln.stride + 1
    tw, th, tn = pick_tile(Wo, Ho)
    halo = (use_halo and not ln.stem and ln.R == 3 and ln.S == 3 and ln.stride == 1 and ln.pad == 1 and Wo >= 8
            and Ho >= 16 and halo_b_stages(P, bn_w, ln.frag_epi) >= 2 and not ln.sparse)
    if halo:
        tw, th, tn = 8, 16, 1
    tiles_w, tiles_h = _ceil(Wo, tw), _ceil(Ho, th)
    if ln.sparse:
        tw, th, tn, tiles_w = Wo, 2, 1, 1
        rows = []
        for i in range(16):
            y0 = int(i * ((Ho - 1) / 15.0))
            if not rows or rows[-1] != y0:
                rows.append(y0)
        tiles_h = len(rows)
    tiles_n = _ceil(ln.N, tn)
    m_tiles = tiles_w * tiles_h * tiles_n
    narrow = has_b64 and (m_tiles * (cout_pad // bn_w) * 2 <= NUM_SMS or max_stages(P, bn_w, ln.frag_epi) < 2)
    cin_blocks = 1 if ln.stem else ln.C // 64
    kb64 = ln.R * ln.S * cin_blocks + (1 if ln.res_mode == 1 and ln.identity else ln.res_C // 64)
    pingpong = (ln.frag_epi and not halo and (bn_w == 64 or has_b64) and max_stages(P, 64, ln.frag_epi) >= 2 and P > 1
                and kb64 <= PINGPONG_MAX_KB)
    block_n = 64 if narrow or pingpong else bn_w
    n_tiles = cout_pad // block_n
    res_kb = 0
    if ln.res_mode == 1 and ln.identity:
        res_kb = block_n // 64
    if ln.res_mode == 4:
        res_kb = ln.res_C // 64
    stages = max_stages(P, block_n, ln.frag_epi)
    if halo:
        stages = 2
    grid = min(m_tiles * n_tiles, NUM_SMS)
    counts = [cta_tiles(m_tiles * n_tiles, b, grid) for b in range(grid)]
    return dict(tw=tw, th=th, tn=tn, tiles_w=tiles_w, tiles_h=tiles_h, tiles_n=tiles_n, block_n=block_n, n_tiles=n_tiles,
                stages=stages, halo=int(halo), res_kb=res_kb, pingpong=int(pingpong), grid=grid,
                cta_tiles_min=min(counts), cta_tiles_max=max(counts), k_blocks=ln.R * ln.S * cin_blocks + res_kb)


def tile_index(total: int, cta: int, grid: int, i: int) -> Optional[int]:
    """gemm_tile_index under schedule 0 (the only schedule outside clusters): the flat tile id, or None."""
    t = cta + i * grid
    return t if t < total else None


def cta_tiles(total: int, cta: int, grid: int) -> int:
    i = 0
    while tile_index(total, cta, grid, i) is not None:
        i += 1
    return i


# ------------------------------------------------------------------------------------------- the protocol
@dataclasses.dataclass
class Faults:
    """Deliberately broken protocols (the model must catch each)."""
    early_handover: bool = False          # the turn is handed over before the tile's last k-block is issued
    skip_last_release: bool = False       # the slot of a tile's last k-block is never released
    empty_count: int = 1                  # readers per empty barrier (2 = as if both warpgroups read every slot)
    turn_without_tile: bool = False       # a warpgroup waits for its next turn before it knows it has a tile


class Mbar:
    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def passed(self, parity):            # mbarrier.try_wait.parity: the phase of this parity has completed
        return (self.phase & 1) != parity


class ProtocolError(Exception):
    pass


def run_protocol(n_tiles: int, nkb: int, stages: int, seed: int = 0, faults: Faults = Faults()) -> Dict[str, object]:
    """One CTA of a ping-pong launch: n_tiles tiles of nkb k-blocks over a `stages`-deep ring, under a random schedule.
    -> {"ok": bool, "error": text or None, "turns": [warpgroup per tile in issue order], "reads": [positions]}"""
    rng = random.Random(seed)
    full = [Mbar(1) for _ in range(stages)]
    empty = [Mbar(faults.empty_count) for _ in range(stages)]
    turn = [Mbar(1), Mbar(1)]
    slot = [None] * stages               # position whose data the slot holds
    tma: List[tuple] = []                # loads in flight: (stage, position)
    groups = {0: [], 1: []}              # wgmma groups in flight per warpgroup: lists of (stage, position)
    reads, turns, filled, released = [], [], [], []

    def has_tile(ti):
        return ti < n_tiles               # tile_at over this CTA's sequence

    def producer():
        st, ph = 0, 0
        for pos in range(n_tiles * nkb):
            yield lambda st=st, ph=ph: empty[st].passed(ph ^ 1)
            tma.append((st, pos))
            filled.append(pos)
            st += 1
            if st == stages:
                st, ph = 0, ph ^ 1

    def consumer(wg):
        ti = wg
        while True:
            if faults.turn_without_tile and ti > 0:
                yield lambda ti=ti: turn[wg].passed(((ti - 1) >> 1) & 1)
            if not has_tile(ti):
                return
            pos0 = ti * nkb
            st, ph = pos0 % stages, (pos0 // stages) & 1
            if ti > 0 and not faults.turn_without_tile:
                yield lambda ti=ti: turn[wg].passed(((ti - 1) >> 1) & 1)
            pend = -1
            for kb in range(nkb):
                if faults.early_handover and kb == nkb - 1:
                    turn[wg ^ 1].arrive()
                yield lambda st=st, ph=ph: full[st].passed(ph)
                pos = pos0 + kb
                if slot[st] != pos:
                    raise ProtocolError(f"warpgroup {wg} read slot {st} for position {pos}, it holds {slot[st]}")
                if kb == 0:
                    turns.append(wg)
                reads.append(pos)
                groups[wg].append((st, pos))
                if kb == nkb - 1 and not faults.early_handover:
                    turn[wg ^ 1].arrive()
                yield lambda: len(groups[wg]) <= 1            # wgmma.wait_group 1
                if pend >= 0:
                    released.append(pend_pos)
                    empty[pend].arrive()
                pend, pend_pos = st, pos
                st += 1
                if st == stages:
                    st, ph = 0, ph ^ 1
            yield lambda: not groups[wg]                      # wgmma.wait_group 0
            if not faults.skip_last_release:
                released.append(pend_pos)
                empty[pend].arrive()
            ti += 2

    agents = {"producer": producer(), "wg0": consumer(0), "wg1": consumer(1)}
    waits = {}
    for name in list(agents):
        try:
            waits[name] = next(agents[name])
        except StopIteration:
            del agents[name]
    try:
        while agents or tma or groups[0] or groups[1]:
            moves = [("agent", n) for n in agents if waits[n]()]
            moves += [("tma", i) for i in range(len(tma))]
            moves += [("wgmma", w) for w in (0, 1) if groups[w]]
            if not moves:
                raise ProtocolError("deadlock: " + ", ".join(sorted(agents)) + " wait forever")
            kind, x = rng.choice(moves)
            if kind == "tma":
                st, pos = tma.pop(x)
                slot[st] = pos
                full[st].arrive()
            elif kind == "wgmma":
                st, pos = groups[x].pop(0)
                if slot[st] != pos:
                    raise ProtocolError(f"slot {st} overwritten while warpgroup {x} read position {pos}")
            else:
                try:
                    waits[x] = next(agents[x])
                except StopIteration:
                    del agents[x]
        total = n_tiles * nkb
        if reads != list(range(total)):
            raise ProtocolError("slots were not read in the producer's order")
        if sorted(filled) != list(range(total)) or sorted(released) != list(range(total)):
            raise ProtocolError("a slot was not filled and released exactly once")
        if turns != [i % 2 for i in range(n_tiles)]:
            raise ProtocolError("turns do not alternate")
    except ProtocolError as e:
        return {"ok": False, "error": str(e), "turns": turns, "reads": reads}
    return {"ok": True, "error": None, "turns": turns, "reads": reads}


def pingpong_schedules(modes=tuple(MODES), batches=(1, 2, 5, 64, 129, 512)):
    """{(tiles in one CTA, k-blocks per tile, ring depth): [launches that run it]} over every ping-pong launch of the plan
    at the given batches and modes (td_parity both ways)."""
    out: Dict[tuple, list] = {}
    for mode in modes:
        P = MODES[mode]
        for B in batches:
            for td in (False, True):
                for ln in network(B, td_parity=td):
                    g = geometry(ln, P)
                    if not g["pingpong"]:
                        continue
                    total = g["tiles_w"] * g["tiles_h"] * g["tiles_n"] * g["n_tiles"]
                    for n in {cta_tiles(total, b, g["grid"]) for b in range(g["grid"])}:
                        out.setdefault((n, g["k_blocks"], g["stages"]), []).append((mode, B, td, ln.layer))
    return out
