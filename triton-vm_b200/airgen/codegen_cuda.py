"""Emit sm_90a CUDA source for the AIR quotient kernels from the lowered constraint circuits.

Reference behaviour being replaced: `all_quotients_combined` (triton-vm/src/table/
master_table.rs:1264-1363) calling the build-time generated `Evaluable::evaluate_*_constraints`
(triton-constraint-builder/src/codegen.rs:59-269).  For every quotient-domain row the result is
    sum_cat  zerofier_inverse_cat(row) * sum_j  weight_j * constraint_j(row, next_row)
with constraint order init | cons | tran | term and, inside a category, base-field-valued
constraints before extension-field-valued ones (codegen.rs:210-212).

Mapping: one thread per row, straight-line code with common sub-expressions shared inside a
chunk.  The 604 constraints are split into many small kernels ("chunks"): a profile of the first
design (14 chunks of ~30k SASS instructions each) showed a low issue rate
with `stalled_no_instruction` dominating - straight-line code that large streams through the
32 KB L1.5 instruction cache once per warp.  A chunk is therefore sized to stay instruction-cache
resident (budget below, ~25 SASS instructions per cost unit); a node needed by two chunks is
recomputed and a chunk re-reads the table columns it touches (on H100 that re-reading is a large part of the stage's HBM
traffic: the degree split below halves it by evaluating every chunk on half of the rows).
Every chunk adds its zerofier-weighted partial sum into the row-planar X-field output.  The
weighted sum  sum_j w_j * c_j  is accumulated UNREDUCED (three 128-bit accumulators + overflow
words, one Montgomery reduction per chunk instead of one per product); the per-weight linear map
a -> a*w is a 3x3 matrix over F_p whose entries are precomputed (7 distinct words per weight).
Weights and challenges live in constant memory (warp-uniform operands).  Chunks are packed into a
few translation units so `make -j` compiles them in parallel.

Run:  python -m airgen.codegen_cuda   (writes csrc/air_gen/*)
"""
import os

from .build import CATEGORIES, build_air
from .circuit import P, reachable_postorder

R = (1 << 64) % P
OUT_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc", "air_gen")
CHUNK_COST_BUDGET = float(os.environ.get("TVM_AIR_BUDGET", "100"))
SYNC_EVERY = int(os.environ.get("TVM_AIR_SYNC_EVERY", "0"))
NUM_TUS = int(os.environ.get("TVM_AIR_TUS", "8"))
MIN_BLOCKS = int(os.environ.get("TVM_AIR_MIN_BLOCKS", "2"))   # __launch_bounds__ minimum blocks per SM of the chunk kernels
# Splitting the few oversized constraints (up to 1079 operations in one kernel) raises the emitted operations by 8-29 %
# (shared sub-expressions are recomputed per piece); with the 128-register cap (MIN_BLOCKS = 2) it pays at 400-cost pieces,
# because the 1 079-operation constraint no longer spills, and not at 250.  On by default at 400.
SPLIT_BIG = os.environ.get("TVM_AIR_SPLIT", "1") != "0"
SPLIT_BUDGET = float(os.environ.get("TVM_AIR_SPLIT_BUDGET", "400"))   # pieces of an oversized constraint may be this large
WTAB_WORDS = 7   # per weight: b0, b1, b2, -b1, -b2, b0+b2, b1-b2
# Degree split: the trace polynomials have degree D < 2n, so the weighted sum of the constraints of degree <= 2 of one zerofier
# class has degree < 4n and is determined by its values on every second coset of the 8n-point quotient domain.  Those
# constraints get their own ("lo") chunks.  When also 3D < 4n, quotient.cu runs the other chunks on half of the rows too and
# corrects the class sums' part of degree >= 4n from the column tops (DESIGN.md section 3); the hi chunks that hold degree-4
# constraints (CHUNK_DEGREE) run once more for that correction.  Exact: same field elements as evaluating everywhere.
DEGREE_SPLIT = os.environ.get("TVM_AIR_DEGREE_SPLIT", "1") != "0"
LOW_DEGREE = 2
CHUNK_CLASS = {}   # chunk index -> "hi" | "lo" (filled by chunk_constraints)
CHUNK_DEGREE = {}  # chunk index -> the largest degree of its constraints (filled by chunk_constraints)


def mont(v):
    return v * R % P


def node_cost(b, n):
    """rough instruction weight of one operation (B-field multiply = 1)"""
    if n.kind not in "+*":
        return 0.0
    lx = not b.evaluates_to_base_element(n.lhs)
    rx = not b.evaluates_to_base_element(n.rhs)
    if n.kind == "*":
        return 9.0 if (lx and rx) else (3.0 if (lx or rx) else 1.0)
    return 1.0 if (lx and rx) else 0.35


# ---- splitting a constraint that is larger than a chunk ------------------------------------------------
# The weighted sum  sum_j w_j c_j  is linear in every c_j, so a constraint may be evaluated as a sum of pieces in
# different kernels (same weight): a top-level sum is cut into groups of terms, and a product `big * small` is
# distributed over the pieces of `big` (small is re-evaluated per piece).  Exact field arithmetic: same value.
# A piece is ("node", n) | ("sum", [pieces]) | ("mul", piece, n).
def subtree_cost(b, n, memo):
    k = id(n)
    if k not in memo:
        memo[k] = sum(node_cost(b, x) for x in reachable_postorder([n]) if x.kind in "+*")
    return memo[k]


def flatten_sum(n):
    out, st = [], [n]
    while st:
        x = st.pop()
        if x.kind == "+":
            st.append(x.rhs); st.append(x.lhs)
        else:
            out.append(x)
    return out


def piece_leaves(piece):
    if piece[0] == "node": return [piece[1]]
    if piece[0] == "sum": return [n for p in piece[1] for n in piece_leaves(p)]
    return piece_leaves(piece[1]) + [piece[2]]


def piece_cost(b, piece):
    return sum(node_cost(b, x) for x in reachable_postorder(piece_leaves(piece)) if x.kind in "+*")


def split_piece(b, n, budget, memo):
    """-> list of pieces whose sum equals node n, each (roughly) within the budget where the shape allows"""
    if subtree_cost(b, n, memo) <= budget or n.kind not in "+*":
        return [("node", n)]
    if n.kind == "+":
        parts = []
        for t in flatten_sum(n):
            parts += split_piece(b, t, budget, memo)
        groups, cur, cur_cost = [], [], 0.0
        for p in parts:
            pc = piece_cost(b, p)
            if cur and cur_cost + pc > budget:
                groups.append(cur); cur, cur_cost = [], 0.0
            cur.append(p); cur_cost += pc
        if cur: groups.append(cur)
        return [g[0] if len(g) == 1 else ("sum", g) for g in groups]
    # product: distribute over the pieces of the expensive factor when the other one is cheap
    cl, cr = subtree_cost(b, n.lhs, memo), subtree_cost(b, n.rhs, memo)
    big, small, cs_ = (n.lhs, n.rhs, cr) if cl >= cr else (n.rhs, n.lhs, cl)
    if cs_ <= budget / 4:
        sub = split_piece(b, big, budget - cs_, memo)
        if len(sub) > 1:
            return [("mul", p, small) for p in sub]
    return [("node", n)]


def chunk_constraints(air, budget=None):
    """-> list of (category, [(global_weight_index, piece)]).  Chunks are runs of the evaluator-order constraint
    list; the budget is in units of B-field multiplications (~18 SASS instructions each): a chunk should stay
    resident in the 32 KB L1.5 instruction cache.  A constraint above the budget is split into pieces."""
    budget = budget or CHUNK_COST_BUDGET
    chunks, offset = [], 0
    for cat in CATEGORIES:
        b = air.builders[cat]
        cs = air.constraints[cat]
        memo = {}
        classes = ("hi", "lo") if DEGREE_SPLIT else ("hi",)
        for cls in classes:
            cur, seen, cost = [], set(), 0.0
            for j, c in enumerate(cs):
                if DEGREE_SPLIT and (b.degree(c) <= LOW_DEGREE) != (cls == "lo"):
                    continue
                pieces = split_piece(b, c, max(budget, SPLIT_BUDGET), memo) if SPLIT_BIG else [("node", c)]
                for piece in pieces:
                    leaves = piece_leaves(piece)
                    new = [x for x in reachable_postorder(leaves) if id(x) not in seen and x.kind in "+*"]
                    new_cost = sum(node_cost(b, x) for x in new) + 6.0
                    if cur and cost + new_cost > budget:
                        CHUNK_CLASS[len(chunks)] = cls
                        CHUNK_DEGREE[len(chunks)] = max(b.degree(cs[i - offset]) for i, _ in cur)
                        chunks.append((cat, cur))
                        cur, seen, cost = [], set(), 0.0
                        new = [x for x in reachable_postorder(leaves) if x.kind in "+*"]
                        new_cost = sum(node_cost(b, x) for x in new) + 6.0
                    cur.append((offset + j, piece))
                    seen.update(id(x) for x in new)
                    cost += new_cost
            if cur:
                CHUNK_CLASS[len(chunks)] = cls
                CHUNK_DEGREE[len(chunks)] = max(b.degree(cs[i - offset]) for i, _ in cur)
                chunks.append((cat, cur))
        offset += len(cs)
    return chunks


class Emitter:
    def __init__(self, builder):
        self.b = builder
        self.lines = []
        self.name = {}       # id(node) -> C expression (variable name or literal)
        self.isx = {}        # id(node) -> bool (X-field valued)
        self.n = 0

    def tmp(self):
        self.n += 1
        return f"t{self.n}"

    def is_neg_one(self, n):
        return n.kind == "B" and n.val == P - 1

    def binop(self, kind, l, r):
        """emit `l kind r` for already emitted operands (name, is_x, is_neg_one) -> (name, is_x)"""
        (ln, lx), (rn, rx) = l, r
        v = self.tmp()
        if kind == "*":
            if lx and rx: expr, resx = f"xmul({ln}, {rn})", True
            elif lx: expr, resx = f"xmulb({ln}, {rn})", True
            elif rx: expr, resx = f"xmulb({rn}, {ln})", True
            else: expr, resx = f"fmul({ln}, {rn})", False
        else:
            if lx and rx: expr, resx = f"xadd({ln}, {rn})", True
            elif lx: expr, resx = f"xaddb({ln}, {rn})", True
            elif rx: expr, resx = f"xaddb({rn}, {ln})", True
            else: expr, resx = f"fadd({ln}, {rn})", False
        self.lines.append(f"const {'xfe' if resx else 'u64'} {v} = {expr};")
        return v, resx

    def emit_piece(self, piece):
        """pieces of a split constraint (see split_piece); leaves are already emitted"""
        if piece[0] == "node":
            n = piece[1]
            return self.name[id(n)], self.isx[id(n)]
        if piece[0] == "sum":
            acc = self.emit_piece(piece[1][0])
            for p in piece[1][1:]:
                acc = self.binop("+", acc, self.emit_piece(p))
            return acc
        inner = self.emit_piece(piece[1])
        n = piece[2]
        return self.binop("*", inner, (self.name[id(n)], self.isx[id(n)]))

    def emit_node(self, n):
        k = n.kind
        key = id(n)
        if k == "B":
            self.name[key] = f"0x{mont(n.val):016x}ULL"; self.isx[key] = False
        elif k == "X":
            v = self.tmp()
            self.lines.append(f"const xfe {v} = xmake(0x{mont(n.val[0]):016x}ULL, 0x{mont(n.val[1]):016x}ULL, 0x{mont(n.val[2]):016x}ULL);")
            self.name[key] = v; self.isx[key] = True
        elif k == "C":
            v = self.tmp()
            i = n.val
            self.lines.append(f"const xfe {v} = xmake(c_ch[{3 * i}], c_ch[{3 * i + 1}], c_ch[{3 * i + 2}]);")
            self.name[key] = v; self.isx[key] = True
        elif k == "I":
            row, is_main, col = n.val
            v = self.tmp()
            if is_main:
                src = "mn" if row else "mc"
                self.lines.append(f"const u64 {v} = {src}[(size_t){col} * a.main_stride];")
                self.isx[key] = False
            else:
                src = "an" if row else "ac"
                self.lines.append(f"const xfe {v} = xmake({src}[(size_t){3 * col} * a.aux_stride], "
                                  f"{src}[(size_t){3 * col + 1} * a.aux_stride], {src}[(size_t){3 * col + 2} * a.aux_stride]);")
                self.isx[key] = True
            self.name[key] = v
        else:
            l, r = n.lhs, n.rhs
            lx, rx = self.isx[id(l)], self.isx[id(r)]
            ln, rn = self.name[id(l)], self.name[id(r)]
            v = self.tmp()
            if k == "*":
                if self.is_neg_one(l) or self.is_neg_one(r):
                    o, ox = (r, rx) if self.is_neg_one(l) else (l, lx)
                    on = self.name[id(o)]
                    expr = f"xneg({on})" if ox else f"fneg({on})"
                    resx = ox
                elif lx and rx: expr, resx = f"xmul({ln}, {rn})", True
                elif lx: expr, resx = f"xmulb({ln}, {rn})", True
                elif rx: expr, resx = f"xmulb({rn}, {ln})", True
                else: expr, resx = f"fmul({ln}, {rn})", False
            else:
                # x + (-1) * y is a subtraction: fsub costs 5 instructions, fneg + fadd 11 (the negation is still emitted
                # above, the compiler drops it when nothing else uses it)
                sub = None
                for pos, neg in ((l, r), (r, l)):
                    if neg.kind == "*" and (self.is_neg_one(neg.lhs) or self.is_neg_one(neg.rhs)):
                        y = neg.rhs if self.is_neg_one(neg.lhs) else neg.lhs
                        px, yx = self.isx[id(pos)], self.isx[id(y)]
                        pn, yn = self.name[id(pos)], self.name[id(y)]
                        if px and yx: sub = (f"xsub({pn}, {yn})", True)
                        elif px: sub = (f"xsubb({pn}, {yn})", True)
                        elif not yx: sub = (f"fsub({pn}, {yn})", False)
                        if sub:
                            break
                if sub: expr, resx = sub
                elif lx and rx: expr, resx = f"xadd({ln}, {rn})", True
                elif lx: expr, resx = f"xaddb({ln}, {rn})", True
                elif rx: expr, resx = f"xaddb({rn}, {ln})", True
                else: expr, resx = f"fadd({ln}, {rn})", False
            self.lines.append(f"const {'xfe' if resx else 'u64'} {v} = {expr};")
            self.name[key] = v; self.isx[key] = resx


TU_HEADER = """// GENERATED by triton-vm_b200/airgen/codegen_cuda.py from the re-derived AIR - do not edit.
// Replaces the build-time generated Evaluable::evaluate_{cat}_constraints of the reference
// (triton-constraint-builder/src/codegen.rs:59-269) fused with the weighted sum and zerofier
// division of all_quotients_combined (triton-vm/src/table/master_table.rs:1264-1363).
#include "../air.cuh"

namespace tvm {
namespace {
__constant__ u64 c_w[%(nw)d];   // weight table of ALL constraints: AIR_WTAB_WORDS words each (see air.cuh)
__constant__ u64 c_ch[189];     // 63 challenges (X-field, Montgomery)
"""

KERNEL_HEADER = """
__global__ void __launch_bounds__(AIR_THREADS, %(minb)d) %(kname)s(AirArgs a) {
  size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
%(guard)s
  const size_t n = (size_t)1 << a.log_n;
  const size_t coset = m >> a.log_n, k = m & (n - 1);
  const size_t mem_base = (coset * a.coset_mem_stride) << a.log_n;
  const size_t m_cur = mem_base | k, m_next = a.next_offset ? m_cur + a.next_offset : mem_base | ((k + 1) & (n - 1));
  const u64 *mc = a.main + m_cur, *mn = a.main + m_next;
  const u64 *ac = a.aux + m_cur, *an = a.aux + m_next;
  (void)mn; (void)an; (void)ac; (void)mc; (void)coset;
"""

BODY_HEADER = """
// constraints %(first)d..%(last)d of the evaluator order (%(cat)s), %(nops)d operations
static __device__ __noinline__ void %(bname)s(const u64 *mc, const u64 *mn, const u64 *ac, const u64 *an, const AirStrides a,
                                              AirAcc &acc_io) {
  (void)mn; (void)an; (void)ac; (void)mc;
"""

TU_FOOTER = """
// `lo` / `hi`: the arguments of the chunks whose constraints have degree <= 2 / up to 4 (see AirArgs::low_out).  A chunk is
// skipped when its group has no rows, or when its largest degree is below the group's min_degree.
void %(tuname)s_launch(const AirArgs &lo, const AirArgs &hi, const u64 *d_wtab, const u64 *d_challenges, cudaStream_t s, unsigned long long *launches) {
  cudaMemcpyToSymbolAsync(c_w, d_wtab, sizeof(u64) * %(nw)d, 0, cudaMemcpyDeviceToDevice, s);
  cudaMemcpyToSymbolAsync(c_ch, d_challenges, sizeof(u64) * 189, 0, cudaMemcpyDeviceToDevice, s);
  const unsigned grid_lo = (unsigned)((lo.nrows + AIR_THREADS - 1) / AIR_THREADS);
  const unsigned grid_hi = (unsigned)((hi.nrows + AIR_THREADS - 1) / AIR_THREADS);
  (void)grid_lo; (void)grid_hi;
  unsigned long long nk = 0;
%(launches)s
  *launches += nk;
}
}  // namespace tvm
"""


def emit_body(air, idx, cat, items, fused):
    """the straight-line code of one chunk: (lines, accumulate lines, #operations)"""
    b = air.builders[cat]
    em = Emitter(b)
    roots = [n for _, piece in items for n in piece_leaves(piece)]
    for n in reachable_postorder(roots):
        em.emit_node(n)
    results = [em.emit_piece(piece) for _, piece in items]
    body = []
    for k, line in enumerate(em.lines):
        body.append(line)
        if not fused and SYNC_EVERY and (k + 1) % SYNC_EVERY == 0:
            body.append("__syncthreads();   // instruction-fetch locality: the CTA's warps share one I-cache window")
    accs = []
    for (j, _), (nm, isx) in zip(items, results):
        accs.append(f"air_acc_{'x' if isx else 'b'}(acc, c_w + {WTAB_WORDS * j}, {nm});")
    nops = sum(1 for n in reachable_postorder(roots) if n.kind in "+*")
    return body, accs, nops


def emit_chunk(air, idx, cat, items):
    body, accs, nops = emit_body(air, idx, cat, items, False)
    low = CHUNK_CLASS.get(idx) == "lo"
    deg = CHUNK_DEGREE[idx]
    kname = f"air_chunk_{idx:03d}_{cat}" + ("_lo" if low else "")
    if SYNC_EVERY:
        guard = "  const bool active = m < a.nrows;\n  if (!active) m = 0;   // keep every thread alive for the block-wide barriers below"
    else:
        guard = "  if (m >= a.nrows) return;\n  const bool active = true;"
    src = [f"\n// constraints of degree <= {deg}" + KERNEL_HEADER % {"kname": kname, "guard": guard, "minb": MIN_BLOCKS}]
    src.append("  " + "\n  ".join(body))
    src.append("  AirAcc acc; air_acc_zero(acc);")
    src.extend("  " + x for x in accs)
    src.append(f"  if (active) air_accumulate_low<{CATEGORIES.index(cat)}>(a, m, coset, air_acc_reduce(acc));")
    src.append("}")
    return kname, "\n".join(src), nops


# ---- fused groups (A/B variant) ---------------------------------------------------------------------------------------
# MEASURED AND REJECTED: chunk kernels at budget 100 beat budget 160 and fused groups of <= 220 or <= 700 cost units.
# A profile of a large group: `stalled_no_instruction` dominates - a group's bodies total 100-300 KB
# of SASS, every CTA streams through all of it once, so the instruction cache misses on every body, and with 174+
# registers there are only 8 warps per SM to hide the fetches.  Kept as an A/B switch (TVM_AIR_FUSED=1); default off.
# One kernel per GROUP of consecutive chunks of a category: the chunk bodies stay separate instruction-cache sized
# functions (`__noinline__`, their own register allocation), the group kernel calls them one after the other on the same
# rows with a block-wide barrier in between, so that (a) the warps of a CTA execute the same body at the same time and
# share one instruction-cache window, (b) the weighted sum is carried across bodies in the unreduced accumulator: one
# reduction, one zerofier multiplication and ONE read-modify-write of the output per group instead of per chunk
# (147 -> ~16 passes over the 3 output planes), (c) columns touched by several bodies of the group are re-read by the
# same CTA right away (L1/L2 hits) instead of by another kernel launch from HBM.  Evaluator order keeps the constraints
# of one table together, so consecutive chunks share their columns.
FUSED = os.environ.get("TVM_AIR_FUSED", "0") != "0"
GROUP_BUDGET = float(os.environ.get("TVM_AIR_GROUP_BUDGET", "700"))


def emit_group(air, gidx, cat, chunk_ids, chunks):
    parts, calls, nops_total = [], [], 0
    for idx in chunk_ids:
        _, items = chunks[idx]
        body, accs, nops = emit_body(air, idx, cat, items, True)
        nops_total += nops
        bname = f"air_body_{idx:03d}_{cat}"
        src = [BODY_HEADER % {"bname": bname, "first": items[0][0], "last": items[-1][0], "cat": cat, "nops": nops}]
        src.append("  " + "\n  ".join(body))
        src.append("  AirAcc acc = acc_io;")
        src.extend("  " + x for x in accs)
        src.append("  acc_io = acc;")
        src.append("}")
        parts.append("\n".join(src))
        calls.append(f"  {bname}(mc, mn, ac, an, st, acc);")
    kname = f"air_group_{gidx:02d}_{cat}"
    guard = "  const bool active = m < a.nrows;\n  if (!active) m = a.nrows - 1;   // every thread takes part in the block-wide barriers below"
    k = [KERNEL_HEADER % {"kname": kname, "guard": guard, "minb": MIN_BLOCKS}]
    k.append("  const AirStrides st{a.main_stride, a.aux_stride};")
    k.append("  AirAcc acc; air_acc_zero(acc);")
    k.append("\n  __syncthreads();   // the CTA's warps share one instruction-cache window\n".join(calls))
    k.append(f"  if (active) air_accumulate_{cat}(a, m, coset, air_acc_reduce(acc));")
    k.append("}")
    parts.append("\n".join(k))
    return kname, "\n".join(parts), nops_total


def group_chunks(air, chunks):
    """consecutive chunks of one category whose estimated cost stays below GROUP_BUDGET"""
    groups, cur, cur_cat, cost = [], [], None, 0.0
    for idx, (cat, items) in enumerate(chunks):
        b = air.builders[cat]
        roots = [n for _, piece in items for n in piece_leaves(piece)]
        c = sum(node_cost(b, x) for x in reachable_postorder(roots) if x.kind in "+*") + 6.0 * len(items)
        if cur and (cat != cur_cat or cost + c > GROUP_BUDGET):
            groups.append((cur_cat, cur))
            cur, cost = [], 0.0
        cur.append(idx); cur_cat = cat; cost += c
    if cur:
        groups.append((cur_cat, cur))
    return groups


def main():
    air = build_air()
    chunks = chunk_constraints(air)
    total_constraints = sum(len(air.constraints[c]) for c in CATEGORIES)
    os.makedirs(OUT_DIR, exist_ok=True)
    for f in os.listdir(OUT_DIR):
        if f != "air_verify_gen.inc":                # written by airgen.codegen_verify
            os.remove(os.path.join(OUT_DIR, f))
    # pack chunks into translation units, balancing the estimated cost (compile time)
    tus = [[] for _ in range(NUM_TUS)]
    load = [0.0] * NUM_TUS
    names, total_ops = [], 0
    if FUSED:
        assert not DEGREE_SPLIT, "the fused-group variant predates the degree split: TVM_AIR_DEGREE_SPLIT=0"
        groups = group_chunks(air, chunks)
        units = {g: emit_group(air, g, cat, ids, chunks) for g, (cat, ids) in enumerate(groups)}
        unit_meta = {g: (cat, sum(len(chunks[i][1]) for i in ids)) for g, (cat, ids) in enumerate(groups)}
    else:
        units = {idx: emit_chunk(air, idx, cat, items) for idx, (cat, items) in enumerate(chunks)}
        unit_meta = {idx: (cat, len(items)) for idx, (cat, items) in enumerate(chunks)}
    order = sorted(units, key=lambda i: -units[i][2])
    for idx in order:
        t = min(range(NUM_TUS), key=lambda i: load[i])
        tus[t].append(idx)
        load[t] += units[idx][2] + 20
    nw = WTAB_WORDS * total_constraints
    tu_names = []
    for t, idxs in enumerate(tus):
        if not idxs:
            continue
        idxs.sort()
        tuname = f"air_tu_{t:02d}"
        tu_names.append(tuname)
        parts = [TU_HEADER % {"nw": nw}, "}  // namespace"]
        launches = []
        for idx in idxs:
            kname, src, nops = units[idx]
            cat, ncons = unit_meta[idx]
            names.append((kname, cat, ncons, nops))
            total_ops += nops
            parts.append(src)
            g = "lo" if kname.endswith("_lo") else "hi"
            deg = 4 if FUSED else CHUNK_DEGREE[idx]
            launches.append(f"  if ({g}.nrows && {g}.min_degree <= {deg}) {{ {kname}<<<grid_{g}, AIR_THREADS, 0, s>>>({g}); nk++; }}")
        parts.append(TU_FOOTER % {"tuname": tuname, "nw": nw, "launches": "\n".join(launches)})
        with open(os.path.join(OUT_DIR, tuname + ".cu"), "w") as f:
            f.write("\n".join(parts))
    unique_ops = sum(sum(1 for n in reachable_postorder(air.constraints[c]) if n.kind in "+*") for c in CATEGORIES)
    with open(os.path.join(OUT_DIR, "air_chunks.inc"), "w") as f:
        f.write("// GENERATED by airgen/codegen_cuda.py - do not edit.\n")
        f.write(f"// {len(names)} {'group' if FUSED else 'chunk'} kernels ({len(chunks)} chunk bodies) in {len(tu_names)} translation units, "
                f"{total_ops} binary operations emitted ({unique_ops} unique in the circuit), chunk budget {CHUNK_COST_BUDGET:g}\n")
        f.write(f"#define TVM_AIR_HAS_LOW_CHUNKS {1 if DEGREE_SPLIT else 0}   // chunks of constraints of degree <= {LOW_DEGREE} carry the suffix _lo\n")
        for tuname in tu_names:
            f.write(f"TVM_AIR_TU({tuname})\n")
        for kname, cat, ncons, nops in sorted(names):
            f.write(f"// {kname}: {ncons} constraints, {nops} ops\n")
    with open(os.path.join(OUT_DIR, "air_meta.inc"), "w") as f:
        f.write("// GENERATED by airgen/codegen_cuda.py - constraint degrees in evaluator order\n")
        f.write("// (the generated *_quotient_degree_bounds of the reference, codegen.rs:222-229).\n")
        for cat in CATEGORIES:
            b = air.builders[cat]
            degs = [b.degree(c) for c in air.constraints[cat]]
            f.write(f"static const int AIR_NUM_{cat.upper()} = {len(degs)};\n")
            f.write(f"static const unsigned char AIR_DEGREES_{cat.upper()}[] = {{{', '.join(map(str, degs))}}};\n")
    print(f"wrote {len(names)} chunks in {len(tu_names)} TUs to {OUT_DIR}: {total_ops} ops emitted, {unique_ops} unique")


if __name__ == "__main__":
    main()
