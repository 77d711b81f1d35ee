"""A seeded corpus of Triton VM programs, one family per instruction group, at the operands where the VM, the table fill and
the AIR branch: u32 operands at 0, 1, 2^31 and 2^32 - 1, field elements at p - 1, RAM pointers that wrap around 0 and
p - 1, Merkle node indices up to 2^32 - 1, jump stacks a thousand deep; random programs that interleave the families
with stack noise; and shape cases that decide which table is the tallest and whether a table has padding rows.

Where it can, a program checks its own results (`<instr> read_io 1 eq assert`): the expected value is computed here with
Python integers (or oracle.field for the extension field, oracle.tip5 for hashes) and passed as public input, so a wrong
result fails inside the VM, not only in a comparison of two VMs.  Test helper, not a test module: `cases()` is the same
list for every call.  Used by tests/test_program_corpus.py (host) and tests/test_zzzzzzz_gpu_program_corpus.py (device)."""
import collections
import functools
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import field as F, tip5, tracegen as tg   # noqa: E402

P = tg.P
U32 = (1 << 32) - 1
SEED = 0x7C0B_2026

Case = collections.namedtuple("Case", "name words public_input secret_input ram digests")

_EDGE_NAMES = {0: "0", 1: "1", 2: "2", 3: "3", 1 << 31: "2^31", U32: "2^32-1", 1 << 32: "2^32", (1 << 32) + 1: "2^32+1",
               1 << 63: "2^63", P - 1: "p-1", P - 2: "p-2", P - 3: "p-3", P - 5: "p-5", 0xAAAAAAAA: "0xAAAAAAAA",
               0x55555555: "0x55555555", 31: "31", 32: "32"}


def vname(v):
    return _EDGE_NAMES.get(v, str(v) if v < 1000 else hex(v))


class Prog:
    """assembly text, public / secret input, initial RAM and secret digests of one program, and a model of the values it
    pushed (the initial 16 stack elements are None: they hold the program digest)"""

    def __init__(self):
        self.src, self.inp, self.sec, self.ram, self.digests = [], [], [], {}, []
        self.st = [None] * 16                    # index 0 = deepest element

    def emit(self, text, delta=0):
        self.src.append(text)
        if delta > 0:
            self.st += [None] * delta
        elif delta < 0:
            del self.st[len(self.st) + delta:]

    def push(self, *vals):
        for v in vals:
            self.src.append(f"push {v % P}")
            self.st.append(v % P)

    def check(self, *vals):
        """the top len(vals) elements are vals, top first (the VM asserts it); pops them"""
        for v in vals:
            self.src.append("read_io 1 eq assert")
            self.inp.append(v % P)
            self.st.pop()

    def check_model(self, k):
        self.check(*[self.st[-1 - i] for i in range(k)])

    def stack_op(self, op, i):
        s = self.st
        if op == "dup":
            s.append(s[-1 - i])
        elif op == "swap":
            s[-1], s[-1 - i] = s[-1 - i], s[-1]
        elif op == "pick":
            s.append(s.pop(len(s) - 1 - i))
        elif op == "place":
            e = s.pop()
            s.insert(len(s) - i, e)
        elif op == "pop":
            del s[len(s) - i:]
        self.src.append(f"{op} {i}")

    def case(self, name):
        return Case(name, tg.assemble(" ".join(self.src + ["halt"])), list(self.inp), list(self.sec), dict(self.ram) or None,
                    [list(d) for d in self.digests])


def _rng(*key):
    return np.random.default_rng([SEED] + [hash_key(k) for k in key])


def hash_key(k):
    return sum(ord(c) << (7 * i % 56) for i, c in enumerate(str(k))) % (1 << 63)


def _u32s(rng, k, top_bit=False):
    v = [int(x) for x in rng.integers(0, 1 << 32, size=k, dtype=np.uint64)]
    return [x | (1 << 31) for x in v] if top_bit else v


def _fes(rng, k):
    return [int(x) for x in rng.integers(0, P, size=k, dtype=np.uint64)]


# ---- u32 families --------------------------------------------------------------------------------------------------
def split_cases():
    rng = _rng("split")
    edges = [0, 1, U32, 1 << 32, (1 << 32) + 1, 1 << 63, P - 2, P - 1]          # p - 1: lo = 0, hi = 2^32 - 1
    out = []
    for k, a in enumerate(edges + _fes(rng, 6)):
        p = Prog()
        p.push(a)
        p.emit("split", 1)
        p.st[-2:] = [a >> 32, a & U32]
        p.check_model(2)
        out.append(p.case(f"split-{vname(a) if k < len(edges) else f'r{k - len(edges)}'}"))
    for k, a in enumerate([0, 5, U32, 1 << 32, P - 1] + _fes(rng, 3) + _u32s(rng, 2)):
        p = Prog()
        p.push(a)
        p.emit("split pop 1 push 0 eq", 0)                    # is_u32: the high half is 0
        p.check(int(a <= U32))
        out.append(p.case(f"is_u32-{vname(a) if k < 5 else f'r{k - 5}'}"))
    return out


def _binary(op, pairs, fn, names):
    out = []
    for (a, b), nm in zip(pairs, names):
        p = Prog()
        p.push(b, a)                                           # a on top
        p.emit(op, -1)
        p.check(fn(a, b))
        out.append(p.case(f"{op}-{nm}"))
    return out


def lt_cases():
    rng = _rng("lt")
    x, y = _u32s(rng, 2)
    pairs = [(0, 0), (x, x), (0, U32), (U32, 0), (U32, U32), (x & ~1, x | 1), (x | 1, x & ~1), (y & ~(1 << 31), y | (1 << 31)),
             (y | (1 << 31), y & ~(1 << 31))]
    names = ["0-0", "x-x", "0-2^32-1", "2^32-1-0", "2^32-1-2^32-1", "bit0-lo-hi", "bit0-hi-lo", "bit31-lo-hi", "bit31-hi-lo"]
    r = _u32s(rng, 12)
    pairs += list(zip(r[:6], r[6:]))
    names += [f"r{k}" for k in range(6)]
    return _binary("lt", pairs, lambda a, b: int(a < b), names)


def bitwise_cases():
    out = []
    for op, fn in (("and", lambda a, b: a & b), ("xor", lambda a, b: a ^ b)):
        rng = _rng(op)
        x = _u32s(rng, 1)[0]
        pairs = [(0, 0), (0, U32), (U32, U32), (0xAAAAAAAA, 0x55555555), (0xAAAAAAAA, 0xAAAAAAAA), (x, x), (U32, x), (x, 0)]
        names = ["0-0", "0-2^32-1", "2^32-1-2^32-1", "0xAAAAAAAA-0x55555555", "0xAAAAAAAA-0xAAAAAAAA", "x-x", "2^32-1-x", "x-0"]
        r = _u32s(rng, 12)
        pairs += list(zip(r[:6], r[6:]))
        names += [f"r{k}" for k in range(6)]
        out += _binary(op, pairs, fn, names)
    return out


def _unary(op, vals, fn, nedge, width=1):
    out = []
    for k, a in enumerate(vals):
        p = Prog()
        p.push(a)
        p.emit(op, width - 1)
        r = fn(a)
        p.check(*(r if isinstance(r, (tuple, list)) else [r]))
        out.append(p.case(f"{op}-{vname(a) if k < nedge else f'r{k - nedge}'}"))
    return out


def log_pop_cases():
    rng = _rng("log_2_floor")
    out = _unary("log_2_floor", [1, 2, 3, 1 << 31, U32] + [max(1, v) for v in _u32s(rng, 5)], lambda a: a.bit_length() - 1, 5)
    return out + _unary("pop_count", [0, 1, 2, 3, 1 << 31, U32] + _u32s(rng, 5), lambda a: bin(a).count("1"), 6)


def pow_cases():
    rng = _rng("pow")
    rb = _fes(rng, 1)[0]
    out = []
    exps = [0, 1, 2, 31, 32, 1 << 31, U32]
    for bn, b in [("0", 0), ("1", 1), ("2", 2), ("2^32-1", U32), ("p-1", P - 1), ("r", rb)]:
        for e in exps:
            p = Prog()
            p.push(e, b)
            p.emit("pow", -1)
            p.check(pow(b, e, P))
            out.append(p.case(f"pow-base={bn}-exp={vname(e)}"))
    for k, (b, e) in enumerate(zip(_fes(rng, 6), _u32s(rng, 6))):
        p = Prog()
        p.push(e, b)
        p.emit("pow", -1)
        p.check(pow(b, e, P))
        out.append(p.case(f"pow-r{k}"))
    return out


def div_mod_cases():
    rng = _rng("div_mod")
    x = _u32s(rng, 1)[0]
    pairs = [(3, 10), (7, 7), (x, 1), (U32, 7), (7, U32), (U32, U32), (0, 5), (U32, 1), (0, U32)]
    names = ["n<d", "n=d", "d=1", "n=2^32-1", "d=2^32-1", "n=d=2^32-1", "n=0", "n=2^32-1-d=1", "n=0-d=2^32-1"]
    r = _u32s(rng, 12)
    pairs += [(a, max(1, b >> (k * 5))) for k, (a, b) in enumerate(zip(r[:6], r[6:]))]
    names += [f"r{k}" for k in range(6)]
    out = []
    for (n, d), nm in zip(pairs, names):
        p = Prog()
        p.push(d, n)
        p.emit("div_mod", 0)
        q, r_ = divmod(n, d)
        p.check(r_, q)
        out.append(p.case(f"div_mod-{nm}"))
    return out


# ---- field, comparison, skiz, extension field --------------------------------------------------------------------------
def field_cases():
    rng = _rng("field")
    out = []
    u, v = _u32s(rng, 2)
    f, g = _fes(rng, 2)
    for (a, b), nm in [((0, 0), "0-0"), ((u, u), "u32-equal"), ((u, u ^ 1), "u32-unequal"), ((P - 1, P - 1), "p-1-p-1"),
                       ((P - 1, P - 2), "p-1-p-2"), ((1 << 32, U32), "2^32-2^32-1"), ((f, f), "field-equal"), ((f, g), "field-unequal")]:
        p = Prog()
        p.push(b, a)
        p.emit("eq", -1)
        p.check(int(a == b))
        out.append(p.case(f"eq-{nm}"))
    for c in (0, 1, P - 1, 1 << 32):
        p = Prog()                                             # skiz over an instruction with an argument
        p.push(10, c)
        p.emit("skiz addi 5", -1)
        p.check(15 if c else 10)
        out.append(p.case(f"skiz-arg-c={vname(c)}"))
        p = Prog()                                             # ... and over one without
        p.push(3, 2, c)
        p.emit("skiz add", -2 if c else -1)
        p.check(5 if c else 2)
        if not c:
            p.emit("pop 1", -1)
        out.append(p.case(f"skiz-noarg-c={vname(c)}"))
    out += _unary("invert", [1, 2, P - 1, P - 2, 1 << 32] + _fes(rng, 4), F.inv, 5)
    for (a, b), nm in [((P - 1, P - 1), "p-1-p-1"), ((1 << 32, 1 << 32), "2^32-2^32"), ((0, P - 1), "0-p-1"), ((f, g), "r0")]:
        p = Prog()
        p.push(a, b)
        p.emit("nop mul", -1)
        p.check(a * b)
        p.push(a, b, a)
        p.emit("add add", -2)
        p.check(2 * a + b)
        out.append(p.case(f"mul-add-{nm}"))
    return out


def _xpush(p, x):
    p.push(x[2], x[1], x[0])


def xfield_cases():
    rng = _rng("xfield")
    r = lambda: tuple(_fes(rng, 3))                              # noqa: E731
    edges = [((1, 0, 0), "1"), ((P - 1, 0, 0), "p-1"), ((0, 1, 0), "0-1-0"), ((0, 0, 1), "0-0-1"), ((0, P - 1, P - 1), "0-p-1-p-1"),
             ((P - 1, P - 1, P - 1), "p-1-p-1-p-1")]
    out = []
    for x, nm in edges + [(r(), f"r{k}") for k in range(4)]:
        p = Prog()
        _xpush(p, x)
        p.emit("x_invert", 0)
        p.check(*F.xinv(x))
        out.append(p.case(f"x_invert-{nm}"))
    pairs = [((0, 0, 0), (1, 2, 3), "zero"), ((1, 0, 0), r(), "one"), ((P - 1, 0, 0), r(), "p-1"), ((0, 1, 0), (0, 1, 0), "x-x"),
             ((0, 0, 1), (0, 0, 1), "x2-x2"), ((P - 1, P - 1, P - 1), (P - 1, P - 1, P - 1), "p-1-all")] + \
        [(r(), r(), f"r{k}") for k in range(4)]
    for x, y, nm in pairs:
        for op, fn in (("xx_mul", F.xmul), ("xx_add", F.xadd)):
            p = Prog()
            _xpush(p, y)
            _xpush(p, x)
            p.emit(op, -3)
            p.check(*fn(x, y))
            out.append(p.case(f"{op}-{nm}"))
        p = Prog()
        _xpush(p, y)
        p.push(x[0])
        p.emit("xb_mul", -1)
        p.check(*F.xmul((x[0], 0, 0), y))
        out.append(p.case(f"xb_mul-{nm}"))
    return out


# ---- RAM -------------------------------------------------------------------------------------------------------------
def _read(p, mem, ptr, k):
    """read_mem k at ptr; checks the returned pointer and the k values"""
    p.push(ptr)
    p.emit(f"read_mem {k}", k)
    p.check((ptr - k) % P, *[mem.get((ptr - j) % P, 0) for j in reversed(range(k))])


def _write(p, mem, ptr, vals):
    """write_mem len(vals) at ptr: vals[0] goes to ptr; checks the returned pointer"""
    for v in reversed(vals):
        p.push(v)
    p.push(ptr)
    p.emit(f"write_mem {len(vals)}", -len(vals))
    for j, v in enumerate(vals):
        mem[(ptr + j) % P] = v % P
    p.check((ptr + len(vals)) % P)


def ram_random_cases():
    out = []
    for k, m in enumerate((10, 20, 30, 40, 50)):
        rng = _rng("ram", k)
        addrs = list(dict.fromkeys([0, 1, P - 2, P - 1] + _fes(rng, m)))
        init = {a: v for a, v in zip(addrs[::2], _fes(rng, len(addrs)))}
        p, mem = Prog(), dict(init)
        p.ram = dict(init)
        order = [addrs[int(i)] for i in rng.permutation(len(addrs))]
        for a in order[: len(order) // 2]:                      # read before write (initial RAM or 0)
            _read(p, mem, a, 1)
        for a in order:                                         # write then read, read twice
            _write(p, mem, a, _fes(rng, 1))
            _read(p, mem, a, 1)
            if int(rng.integers(0, 3)) == 0:
                _read(p, mem, a, 1)
        for a in order[::3]:                                    # overwrite
            _write(p, mem, a, _fes(rng, 1))
        for i in rng.permutation(len(addrs)):                   # read back shuffled
            _read(p, mem, addrs[int(i)], 1)
        out.append(p.case(f"ram_random-{m}-addresses"))
    return out


def ram_wrap_cases():
    out = []
    rng = _rng("ram_wrap")
    for op in ("read_mem", "write_mem"):
        for a in (0, 1, 3, P - 1, P - 3):
            init = {(a + d) % P: v for d, v in zip(range(-6, 7), _fes(rng, 13))}
            p, mem = Prog(), dict(init)
            p.ram = dict(init)
            for k in range(1, 6):
                if op == "read_mem":
                    _read(p, mem, a, k)
                else:
                    _write(p, mem, a, _fes(rng, k))
                    _read(p, mem, (a + k - 1) % P, k)
            out.append(p.case(f"ram_wrap-{op}-at={vname(a)}"))
    for a in (P - 5, P - 1, 0):
        init = {(a + d) % P: v for d, v in zip(range(10), _fes(rng, 10))}
        p = Prog()
        p.ram = dict(init)
        p.emit("sponge_init")
        p.push(0, 0, 0, 0, a)
        p.emit("sponge_absorb_mem", 0)
        vals = [init[(a + d) % P] for d in range(10)]
        p.check((a + 10) % P, *vals[:4])
        state = tip5.permutation(vals + [0] * 6)
        p.emit("sponge_squeeze", 10)
        p.check(*state[:10])
        out.append(p.case(f"ram_wrap-sponge_absorb_mem-at={vname(a)}"))
    for op, width in (("b_horner_step", 1), ("x_horner_step", 3)):
        for a in (0, 1, 2):
            out.append(_horner(op, width, a, 3, rng, f"ram_wrap-{op}-at={a}"))
    return out


def _horner(op, width, a, steps, rng, name):
    """`steps` Horner steps from pointer a (RAM: coefficients at a, a - 1, ...); checks the pointer and the accumulator"""
    init = {(a - d) % P: v for d, v in zip(range(width * steps), _fes(rng, width * steps))}
    x, acc = tuple(_fes(rng, 3)), tuple(_fes(rng, 3))
    p = Prog()
    p.ram = dict(init)
    p.push(acc[2], acc[1], acc[0], 0, a, 0, 0, x[2], x[1], x[0])
    ptr = a
    for _ in range(steps):
        p.emit(op)
        if width == 1:
            c = (init[ptr], 0, 0)
        else:
            c = (init[(ptr - 2) % P], init[(ptr - 1) % P], init[ptr])
        acc = F.xadd(F.xmul(acc, x), c)
        ptr = (ptr - width) % P
    p.emit("pop 5", -5)
    p.check(ptr, 0, *acc)
    return p.case(name)


def horner_merkle_cases():
    out = []
    for k in range(2):
        rng = _rng("horner", k)
        a = _fes(rng, 1)[0]
        out.append(_horner("b_horner_step", 1, a, 9, rng, f"horner-b_horner_step-r{k}"))
        out.append(_horner("x_horner_step", 3, a, 6, rng, f"horner-x_horner_step-r{k}"))
    for mem in (False, True):
        for idx in (1, 2, 3, U32):
            rng = _rng("merkle", mem, idx)
            leaf = _fes(rng, 5)
            depth = max(1, idx.bit_length())
            sibs = [_fes(rng, 5) for _ in range(depth)]
            p = Prog()
            ptr = _fes(rng, 1)[0]
            if mem:
                p.ram = {(ptr + 5 * j + i) % P: s[i] for j, s in enumerate(sibs) for i in range(5)}
                p.push(ptr, 0)
            else:
                p.digests = sibs
            p.push(idx, *reversed(leaf))
            cur, i = leaf, idx
            for s in sibs:
                p.emit("merkle_step_mem" if mem else "merkle_step")
                cur = [int(v) for v in (tip5.hash_pair(cur, s) if i % 2 == 0 else tip5.hash_pair(s, cur))]
                i //= 2
            p.check(*cur, i)
            if mem:
                p.check(0, (ptr + 5 * depth) % P)
            out.append(p.case(f"merkle-{'merkle_step_mem' if mem else 'merkle_step'}-index={vname(idx)}-depth={depth}"))
    return out


def hash_cases():
    out = []
    for v, nm in ((0, "0"), (P - 1, "p-1")):
        p = Prog()
        p.push(*[v] * 10)
        p.emit("hash", -5)
        digest = [int(x) for x in tip5.hash_10([v] * 10)]
        p.emit("read_io 5 assert_vector", 0)                     # st0..4 against the input, reversed
        p.inp += list(reversed(digest))
        p.check(*digest)
        out.append(p.case(f"hash-all-{nm}"))
    for k in range(3):
        rng = _rng("sponge", k)
        p = Prog()
        p.emit("sponge_init")
        state = [0] * 16
        ptr = [0, P - 10, _fes(rng, 1)[0]][k]
        p.ram = {(ptr + i) % P: v for i, v in enumerate(_fes(rng, 30))}
        p.push(0, 0, 0, 0, ptr)
        for step in "a m s a s m m s".split():
            if step == "a":                                    # sponge_absorb of 10 words; st0 goes to state[0]
                vals = _fes(rng, 10)
                p.push(*reversed(vals))
                p.emit("sponge_absorb", -10)
                state = tip5.permutation(vals + state[10:])
            elif step == "m":                                  # sponge_absorb_mem at the pointer on top
                vals = [p.ram.get((ptr + i) % P, 0) for i in range(10)]
                p.emit("sponge_absorb_mem", 0)
                ptr = (ptr + 10) % P
                state = tip5.permutation(vals + state[10:])
            else:
                p.emit("sponge_squeeze", 10)
                p.check(*state[:10])
                state = tip5.permutation(state)
        p.check(ptr)
        out.append(p.case(f"sponge-r{k}"))
    return out


# ---- stack and control flow ---------------------------------------------------------------------------------------------
def stack_cases():
    out = []
    for op in ("dup", "swap", "pick", "place"):
        rng = _rng("stack", op)
        p = Prog()
        p.push(*_fes(rng, 20))
        for i in range(16):
            p.stack_op(op, i)
            p.emit("dup 0", 1); p.st[-1] = p.st[-2]
            p.check_model(1)
        for i in range(15, -1, -1):
            p.stack_op(op, i)
        p.check_model(16)
        out.append(p.case(f"stack-{op}-0..15"))
    rng = _rng("stack", "words")
    p = Prog()
    for k in range(1, 6):
        vals = _fes(rng, k)
        p.sec += vals
        p.emit(f"divine {k}", k)
        p.st[-k:] = vals
        p.check_model(k)
        vals = _fes(rng, k)
        p.inp += vals
        p.emit(f"read_io {k}", k)
        p.st[-k:] = vals
        p.emit(f"write_io {k}", -k)
        p.push(*_fes(rng, k))
        p.stack_op("pop", k)
        mem = {}
        _write(p, mem, 1000 * k, _fes(rng, k))
        _read(p, mem, 1000 * k + k - 1, k)
    out.append(p.case("stack-word-arguments-1..5"))
    rng = _rng("stack", "deep")
    p = Prog()                                                  # 1500 elements deep and back
    vals = _fes(rng, 1500)
    p.sec += vals
    p.emit("divine 5 " * 300, 1500)
    p.st[-1500:] = vals                                          # each divine pushes its words in order
    for op, i in (("dup", 15), ("dup", 15), ("swap", 15), ("pick", 15), ("place", 15), ("pick", 7), ("pop", 2)):
        p.stack_op(op, i)
    p.check_model(3)
    p.emit("pop 5 " * 299, -1495)
    p.emit("pop 2", -2)
    out.append(p.case("stack-1500-deep"))
    return out


def _call_program(depth, loop):
    """a recursion `depth` calls deep (jump stack depth + 1), a `recurse` loop and a `recurse_or_return` loop of `loop`
    iterations each, under an outer call"""
    return f"""
        call main
        halt
        main:
            push {depth} call rec pop 1
            push {loop} call count_down pop 1
            push {loop} push 0 push 0 push 0 push 0 push 0 push 0 call ror pop 5 pop 2
            return
        rec:        addi -1 dup 0 skiz call rec return
        count_down: addi -1 dup 0 push 0 eq skiz return recurse
        ror:        swap 5 addi 1 swap 5 recurse_or_return
    """


def control_cases():
    p = Prog()
    p.src.append(_call_program(300, 60).replace("halt", "push 1 read_io 1 eq assert halt", 1))
    p.inp.append(1)
    words = tg.assemble(" ".join(p.src))
    return [Case("control-jump-stack-301-deep", words, [1], [], None, [])]


# ---- random programs -------------------------------------------------------------------------------------------------------
def random_program(seed, length):
    """-> Case: about `length` instructions of self-contained snippets from every family, interleaved with stack noise.
    Only the stack depth is tracked; each snippet pushes its own operands, so u32 operands, divisors and inverses are valid."""
    rng = np.random.default_rng([SEED, 0x5EED, seed])
    p = Prog()
    pool = list(dict.fromkeys([0, 1, P - 2, P - 1] + _fes(rng, 6)))
    p.ram = {a: v for a, v in zip(pool[1::2], _fes(rng, len(pool)))}
    mem = dict(p.ram)
    p.emit("sponge_init")
    count = 0

    def depth():
        return len(p.st)

    def fill_to(d):
        while depth() < d:
            p.push(_fes(rng, 1)[0])

    def u32(top_bit=False):
        v = _u32s(rng, 1, top_bit)[0]
        return [0, 1, U32, v, v][int(rng.integers(0, 5))]

    snippets = ["lt", "and", "xor", "log", "popc", "pow", "div", "split", "eq", "inv", "xinv", "xmul", "xbmul", "xadd", "read",
                "write", "hash", "absorb", "squeeze", "absorb_mem", "merkle", "merkle_mem", "bhorner", "xhorner", "call", "skiz",
                "divine", "write_io", "noise", "noise", "noise", "noise"]
    while count < length:
        s = snippets[int(rng.integers(0, len(snippets)))]
        before = len(p.src)
        if s in ("lt", "and", "xor"):
            a, b = u32(True), u32()
            if rng.integers(0, 2):
                a, b = b, a
            p.push(b, a)
            p.emit(s, -1)
            p.check({"lt": int(a < b), "and": a & b, "xor": a ^ b}[s])
        elif s == "log":
            a = max(1, u32())
            p.push(a); p.emit("log_2_floor"); p.check(a.bit_length() - 1)
        elif s == "popc":
            a = u32()
            p.push(a); p.emit("pop_count"); p.check(bin(a).count("1"))
        elif s == "pow":
            b, e = [0, 1, P - 1, _fes(rng, 1)[0]][int(rng.integers(0, 4))], u32()
            p.push(e, b); p.emit("pow", -1); p.check(pow(b, e, P))
        elif s == "div":
            n, d = u32(), max(1, u32() >> int(rng.integers(0, 32)))
            p.push(d, n); p.emit("div_mod"); p.check(n % d, n // d)
        elif s == "split":
            a = _fes(rng, 1)[0]
            p.push(a); p.emit("split", 1); p.check(a & U32, a >> 32)
        elif s == "eq":
            a = _fes(rng, 1)[0]
            b = a if rng.integers(0, 2) else _fes(rng, 1)[0]
            p.push(b, a); p.emit("eq", -1); p.check(int(a == b))
        elif s == "inv":
            a = max(1, _fes(rng, 1)[0])
            p.push(a); p.emit("invert"); p.check(F.inv(a))
        elif s == "xinv":
            x = tuple(_fes(rng, 3))
            _xpush(p, x); p.emit("x_invert"); p.check(*F.xinv(x))
        elif s in ("xmul", "xadd"):
            x, y = tuple(_fes(rng, 3)), tuple(_fes(rng, 3))
            _xpush(p, y); _xpush(p, x); p.emit("xx_mul" if s == "xmul" else "xx_add", -3)
            p.check(*(F.xmul(x, y) if s == "xmul" else F.xadd(x, y)))
        elif s == "xbmul":
            y, c = tuple(_fes(rng, 3)), _fes(rng, 1)[0]
            _xpush(p, y); p.push(c); p.emit("xb_mul", -1); p.check(*F.xmul((c, 0, 0), y))
        elif s == "read":
            _read(p, mem, pool[int(rng.integers(0, len(pool)))], int(rng.integers(1, 6)))
        elif s == "write":
            _write(p, mem, pool[int(rng.integers(0, len(pool)))], _fes(rng, int(rng.integers(1, 6))))
        elif s == "hash":
            fill_to(26); p.emit("hash", -5)
        elif s == "absorb":
            fill_to(26); p.emit("sponge_absorb", -10)
        elif s == "squeeze":
            p.emit("sponge_squeeze", 10)
        elif s == "absorb_mem":
            p.push(pool[int(rng.integers(0, len(pool)))]); p.emit("sponge_absorb_mem"); p.emit("pop 1", -1)
        elif s in ("merkle", "merkle_mem"):
            if s == "merkle_mem":
                p.push(pool[int(rng.integers(0, len(pool)))], 0)
            else:
                p.digests.append(_fes(rng, 5))
            p.push(u32(), *_fes(rng, 5))
            p.emit("merkle_step" if s == "merkle" else "merkle_step_mem")
            p.emit("pop 5 pop 3" if s == "merkle_mem" else "pop 5 pop 1", -8 if s == "merkle_mem" else -6)
        elif s in ("bhorner", "xhorner"):
            p.emit("b_horner_step" if s == "bhorner" else "x_horner_step")
        elif s == "call":
            a = _fes(rng, 1)[0]
            p.push(a); p.emit("call add7 call square"); p.check((a + 7) ** 2)
        elif s == "skiz":
            c = [0, 1, _fes(rng, 1)[0]][int(rng.integers(0, 3))]
            p.push(10, c); p.emit("skiz addi 5", -1); p.check(15 if c else 10)
        elif s == "divine":
            k = int(rng.integers(1, 6))
            vals = _fes(rng, k)
            p.sec += vals
            p.emit(f"divine {k}", k)
            p.st[-k:] = vals
            p.check_model(k)
        elif s == "write_io":
            k = int(rng.integers(1, 6))
            fill_to(16 + k); p.emit(f"write_io {k}", -k)
        else:
            op = ["dup", "swap", "pick", "place", "push", "pop"][int(rng.integers(0, 6))]
            if op == "push":
                p.push(_fes(rng, 1)[0])
            elif op == "pop":
                k = int(rng.integers(1, 6))
                fill_to(16 + k); p.stack_op("pop", k)
            elif op == "dup":
                p.stack_op("dup", int(rng.integers(0, 16)))
            else:
                fill_to(17)                                     # place pops the top first
                p.stack_op(op, int(rng.integers(0, 16)))
        if depth() > 60:
            p.stack_op("pop", 5)
        count += sum(len(t.split()) for t in p.src[before:]) // 2 + 1
    p.src.append("halt add7: addi 7 return square: dup 0 mul return")
    words = tg.assemble(" ".join(p.src))
    return Case(f"random-seed={seed}", words, list(p.inp), list(p.sec), dict(p.ram), [list(d) for d in p.digests])


# ---- shape cases ------------------------------------------------------------------------------------------------------------
# Loops, not straight-line code: the program hash feeds the cascade table, and a long program would make it the tallest.
_LOOP_TAIL = "swap 10 addi -1 swap 10 dup 10 push 0 eq skiz return recurse"      # counter at st10


def shape_cases():
    out = []
    rng = _rng("shape")
    # u32 dominated: 170 iterations of and / lt / pow on a counter a >= 2^31, three 33-row sections each, 16 830 u32 rows
    p = Prog()
    p.push(170, *_fes(rng, 9), 1 << 31)
    p.src.append("call body pop 5 pop 5 pop 1 halt body: addi 1 dup 0 push 4294967295 and pop 1 dup 0 push 4294967295 lt pop 1 "
                 "dup 0 push 3 pow pop 1 " + _LOOP_TAIL)
    out.append(Case("shape-u32-dominated", tg.assemble(" ".join(p.src)), [], [], None, []))
    # a u32 table of exactly 2^12 rows: 124 sections of 33 rows and one of 4, no padding rows
    p = Prog()
    p.push(124, *_fes(rng, 9), 1 << 31)
    p.src.append("call body pop 5 pop 5 pop 1 push 1 push 5 lt pop 1 halt body: addi 1 dup 0 push 4294967295 and pop 1 " + _LOOP_TAIL)
    out.append(Case("shape-u32-exactly-2^12", tg.assemble(" ".join(p.src)), [], [], None, []))
    # RAM dominated: runs of 8 x_horner_step (24 consecutive pointers) at 400 bases drawn from the whole field (secret
    # input), 9 600 unique pointers: the two-pass Bezout transforms
    bases = _fes(rng, 400)
    ram = {(b - d) % P: v for b in bases[::3] for d, v in zip(range(24), _fes(rng, 24))}
    src = ("push 400 " + " ".join(f"push {v}" for v in _fes(rng, 10)) + " call body halt "
           "body: swap 5 pop 1 divine 1 swap 5 " + "x_horner_step " * 8 + _LOOP_TAIL)
    out.append(Case("shape-ram-dominated", tg.assemble(src), [], bases, ram, []))
    # hash dominated: sponge_absorb_mem at one pointer and merkle_step at node index 0 write no op-stack rows; the hash table
    # is taller than the processor, RAM and op-stack tables (the cascade table, fed by the same permutations, is the tallest)
    ptr = _fes(rng, 1)[0]
    src = (f"sponge_init push 150 push 0 push 0 push 0 push 0 push 0 push 0 push 0 push 0 push 0 push {ptr} call body halt "
           "body: sponge_absorb_mem addi -10 swap 6 merkle_step merkle_step merkle_step swap 6 " + _LOOP_TAIL)
    out.append(Case("shape-hash-dominated", tg.assemble(src), [], [], {(ptr + i) % P: v for i, v in enumerate(_fes(rng, 10))},
                    [_fes(rng, 5) for _ in range(450)]))
    # op-stack dominated: a recursion 400 deep that divines 5 words per level, 2 000 elements deep and back (400 words of output)
    src = ("push 400 call deep halt "
           "deep: divine 5 pick 5 addi -1 dup 0 skiz call deep addi 1 place 5 write_io 1 pop 4 return")
    out.append(Case("shape-op-stack-dominated", tg.assemble(src), [], _fes(rng, 2000), None, []))
    # a processor trace of exactly 2^13 rows (processor and jump-stack tables without padding rows), a jump stack 1001 deep
    rows = lambda loop: len(tg.execute(tg.assemble(_call_program(1000, loop))).rows)      # noqa: E731
    r1, step = rows(1), rows(2) - rows(1)
    loop = 1 + ((1 << 13) - r1) // step
    words = tg.assemble("nop " * ((1 << 13) - rows(loop)) + _call_program(1000, loop))
    out.append(Case("shape-processor-exactly-2^13", words, [], [], None, []))
    return out


# ---- the corpus -----------------------------------------------------------------------------------------------------------
FAMILIES = (split_cases, lt_cases, bitwise_cases, log_pop_cases, pow_cases, div_mod_cases, field_cases, xfield_cases,
            ram_random_cases, ram_wrap_cases, horner_merkle_cases, hash_cases, stack_cases, control_cases)
RANDOM_SEEDS = range(20)
RANDOM_LENGTH = 200


@functools.lru_cache(maxsize=None)
def _all():
    out = [c for fam in FAMILIES for c in fam()]
    out += [random_program(s, RANDOM_LENGTH) for s in RANDOM_SEEDS]
    out += shape_cases()
    names = [c.name for c in out]
    assert len(set(names)) == len(names), [n for n in names if names.count(n) > 1]
    return tuple(out)


def cases():
    """-> [Case(name, words, public_input, secret_input, ram, digests)], the same list for every call"""
    return list(_all())


def by_name(name):
    return next(c for c in _all() if c.name == name)
