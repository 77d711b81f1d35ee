"""Constraints::all() + degree lowering — restates triton-constraint-builder/src/lib.rs:38-184
and the build script triton-vm/build.rs:11-25.

`build_air()` returns, per category (init, cons, tran, term):
  * the final constraint list in evaluator order: originals ++ main substitutions ++ aux
    substitutions (lib.rs:174-184), then stably partitioned base-field-valued first
    (codegen.rs:210-212, 243-252);
  * the substitution rules, from which the derived (degree-lowering) columns are filled
    (substitutions.rs:128-301);
  * the origin of every constraint, in a list parallel to the constraint list: (ORIGIN_* index, origin index), where the
    origin index of an original constraint is its position in its table's list for that category before lowering (the
    `idx` of the reference's ConstraintError, stark.rs:2899-3015), and that of a substitution constraint the derived
    column it defines (main 149..378 or aux 49..89).
"""
import time

from . import cross_table
from .circuit import Builder, lower_to_degree, num_visible_nodes, multicircuit_degree
from .columns import NUM_MAIN_COLUMNS, NUM_AUX_COLUMNS
from .tables import program, processor, op_stack, ram, jump_stack, hash, cascade, lookup, u32

TARGET_DEGREE = 4            # triton-air/src/lib.rs:37
PROVIDERS = [program, processor, op_stack, ram, jump_stack, hash, cascade, lookup, u32, cross_table]
CATEGORIES = ["init", "cons", "tran", "term"]
_FN = {"init": "initial", "cons": "consistency", "tran": "transition", "term": "terminal"}
# origins of a constraint: the nine tables in MasterMainTable order (= PROVIDERS), the Grand Cross-Table Argument, and
# the degree lowering, whose substitution constraints define the derived main / aux columns
ORIGIN_NAMES = ["ProgramTable", "ProcessorTable", "OpStackTable", "RamTable", "JumpStackTable", "HashTable", "CascadeTable",
                "LookupTable", "U32Table", "GrandCrossTableArg", "DegreeLowering"]
ORIGIN_DEGREE_LOWERING = len(ORIGIN_NAMES) - 1

# specification/src/arithmetization-overview.md:28-78
EXPECTED_BEFORE = {"init": (79, 539), "cons": (79, 637), "tran": (152, 6825), "term": (23, 213)}
EXPECTED_AFTER = {"init": (81, 543), "cons": (97, 689), "tran": (403, 7400), "term": (23, 213)}


class Air:
    pass


def build_air(verbose=False):
    air = Air()
    air.builders, air.roots, air.before = {}, {}, {}
    root_origins = {}
    for cat in CATEGORIES:
        b = Builder(dual=(cat == "tran"))
        roots, root_origins[cat] = [], []
        for k, prov in enumerate(PROVIDERS):
            cs = [m.n for m in getattr(prov, _FN[cat])(b)]
            roots += cs
            root_origins[cat] += [(k, j) for j in range(len(cs))]
        air.builders[cat], air.roots[cat] = b, roots
        air.before[cat] = (len(roots), num_visible_nodes(roots), multicircuit_degree(b, roots))
        if verbose:
            print(cat, "before lowering: constraints, nodes, degree =", air.before[cat], flush=True)
    # lower_to_target_degree_through_substitutions (lib.rs:131-171): column counters carry over
    n_main, n_aux = NUM_MAIN_COLUMNS, NUM_AUX_COLUMNS
    air.main_subst, air.aux_subst, air.after, air.constraints = {}, {}, {}, {}
    air.subst_col_start, air.origins = {}, {}
    for cat in CATEGORIES:
        t0 = time.time()
        b, roots = air.builders[cat], air.roots[cat]
        air.subst_col_start[cat] = (n_main, n_aux)
        ms, xs = lower_to_degree(b, roots, TARGET_DEGREE, n_main, n_aux)
        n_main += len(ms); n_aux += len(xs)
        air.main_subst[cat], air.aux_subst[cat] = ms, xs
        allc = roots + ms + xs
        air.after[cat] = (len(allc), num_visible_nodes(allc), multicircuit_degree(b, allc))
        origins = root_origins[cat] + [(ORIGIN_DEGREE_LOWERING, n_main - len(ms) + k) for k in range(len(ms))] + \
            [(ORIGIN_DEGREE_LOWERING, n_aux - len(xs) + k) for k in range(len(xs))]
        # the partition goes by position: deduplicated nodes may stand at several positions
        is_base = [b.evaluates_to_base_element(c) for c in allc]
        order = [i for i in range(len(allc)) if is_base[i]] + [i for i in range(len(allc)) if not is_base[i]]
        air.constraints[cat] = [allc[i] for i in order]
        air.origins[cat] = [origins[i] for i in order]
        if verbose:
            print(cat, "after lowering:", air.after[cat], f"(+{len(ms)} main, +{len(xs)} aux columns)",
                  f"{time.time() - t0:.1f}s", flush=True)
    air.num_main_columns, air.num_aux_columns = n_main, n_aux
    return air


if __name__ == "__main__":
    a = build_air(verbose=True)
    print("main columns", a.num_main_columns, "aux columns", a.num_aux_columns)
    for cat in CATEGORIES:
        print(cat, "before ok" if a.before[cat][:2] == EXPECTED_BEFORE[cat] else f"BEFORE MISMATCH {EXPECTED_BEFORE[cat]}",
              "| after ok" if a.after[cat][:2] == EXPECTED_AFTER[cat] else f"| AFTER MISMATCH {EXPECTED_AFTER[cat]}")
