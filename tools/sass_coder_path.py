"""Development tool (CPU only): the range coder's matched path in the SASS of every k_entropy instance.

    python tools/sass_coder_path.py [OBJ_OR_SO] [--list]

OBJ_OR_SO defaults to cool-chic_b200/csrc/ccd_entropy.o (cuobjdump -sass reads a .o, a .so or a cubin).

A speculative round ends with the record read-back: an LDS.128 of (D, R) followed by an LDS.64 of (words consumed,
tag) 16 bytes further.  From each read-back the tool follows the shortest path (in instructions) to the next
read-back that makes no unpredicated CALL: the matched round, where every rare case stays behind a branch that is
not taken or a predicated call that does not fire.  It prints, per read-back, the instructions on that path, its
taken branches (with their kinds) and any LDL / STL; --list prints the path itself.

DESIGN §4.1 wants at most one taken branch per two rounds on that path (the back-edge) and no local memory.
"""
import heapq
import os
import re
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DIVERGED = 100000  # a converged warp never takes BRA.DIV: its target is off any real path
INS = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def functions(path):
    out = subprocess.run(["cuobjdump", "-sass", path], check=True, capture_output=True, text=True).stdout
    name, body = None, []
    for line in out.splitlines():
        if "Function :" in line:
            if name:
                yield name, body
            name, body = line.split("Function :")[1].strip(), []
            continue
        m = INS.match(line)
        if m and name:
            body.append((int(m.group(1), 16), m.group(2)))
    if name:
        yield name, body


def demangle(name):
    m = re.search(r"k_entropyILi(\d+)ELi(\d+)ELb([01])E", name)
    return f"k_entropy<{m.group(1)}, {m.group(2)}, {'true' if m.group(3) == '1' else 'false'}>" if m else name


def parse(text):
    """(predicate or None, opcode, operands)"""
    pred = None
    if text.startswith("@"):
        pred, text = text.split(None, 1)
    parts = text.split(None, 1)
    return pred, parts[0], parts[1] if len(parts) > 1 else ""


def mem_operand(ops):
    m = re.search(r"\[(R\d+|RZ)(?:\+(0x[0-9a-f]+))?\]", ops)
    return (m.group(1), int(m.group(2) or "0", 16)) if m else None


def record_loads(body):
    """indices of LDS.128 [X+o] followed within three instructions by LDS.64 [X+o+16]"""
    idx = []
    for i, (_, t) in enumerate(body):
        _, op, ops = parse(t)
        if op != "LDS.128":
            continue
        a = mem_operand(ops)
        for k in range(i + 1, min(i + 4, len(body))):
            _, op2, ops2 = parse(body[k][1])
            if op2 == "LDS.64" and a and mem_operand(ops2) == (a[0], a[1] + 16):
                idx.append(i)
                break
    return idx


def successors(body, at, i):
    """[(j, taken, kind)] of instruction i; kind names a taken edge"""
    pred, op, ops = parse(body[i][1])
    conditional = pred not in (None, "@PT")
    nxt = [(i + 1, False, None)] if i + 1 < len(body) else []
    if op.startswith("BRA") or op.startswith("JMP"):
        m = re.findall(r"0x([0-9a-f]+)", ops)
        tgt = at.get(int(m[-1], 16)) if m else None
        if re.match(r"^!?U?P\d+,", ops) or op == "BRA.DIV":
            conditional = True  # BRA P2, target: a predicate operand; BRA.DIV: taken only by a diverged warp
        t = [(tgt, True, ("cond " if conditional else "") + op)] if tgt is not None else []
        if tgt == i + 1:
            t = [(tgt, False, None)]
        return t + (nxt if conditional else [])
    if op in ("EXIT", "RET", "RET.REL", "RET.REL.NODEC", "BRX", "JMX") or op.startswith("RET") or op.startswith("BRX"):
        return nxt if conditional else []
    if op.startswith("CALL") and not conditional:
        return []  # an unconditional call leaves the matched path
    return nxt


def matched_path(body, at, start, stops):
    """shortest path start -> (a record load other than start, or start itself around the loop)"""
    dist = {start: 0}
    prev = {}
    heap = [(0, start)]
    while heap:
        d, i = heapq.heappop(heap)
        if d > dist.get(i, 1 << 30):
            continue
        if i != start and i in stops:
            path = [i]
            while path[-1] != start:
                path.append(prev[path[-1]][0])
            path.reverse()
            edges = [prev[p] for p in path[1:]]
            return path, edges
        for j, taken, kind in successors(body, at, i):
            if j is None:
                continue
            nd = d + (DIVERGED if kind == "cond BRA.DIV" else 1)
            if nd < dist.get(j, 1 << 30):
                dist[j] = nd
                prev[j] = (i, taken, kind)
                heapq.heappush(heap, (nd, j))
    return None, None


def report(path, listing):
    for name, body in functions(path):
        if "k_entropy" not in name:
            continue
        at = {a: i for i, (a, _) in enumerate(body)}
        recs = record_loads(body)
        print(f"{demangle(name)}: {len(body)} instructions, {len(recs)} record read-backs")
        for r in recs:
            p, edges = matched_path(body, at, r, set(recs))
            if p is None:
                print(f"  {body[r][0]:#07x}: no call-free path to a record read-back")
                continue
            taken = [(body[e[0]][0], e[2]) for e in edges if e[1]]
            local = [body[i][1] for i in p[:-1] if parse(body[i][1])[1].split(".")[0] in ("LDL", "STL")]
            pcalls = [body[i][0] for i in p[:-1] if parse(body[i][1])[1].startswith("CALL")]
            pbra = [body[i][0] for i in p[:-1] if parse(body[i][1])[1] == "BRA" and (i, True) not in
                    [(e[0], e[1]) for e in edges]]
            ndiv = sum(parse(body[i][1])[1] == "BRA.DIV" for i in p[:-1])
            print(f"  {body[r][0]:#07x} -> {body[p[-1]][0]:#07x}: {len(p) - 1} instructions, "
                  f"{len(taken)} taken branch(es) {['%#x %s' % t for t in taken]}, "
                  f"{len(pbra)} branch(es) not taken, {len(pcalls)} predicated call(s) not taken, {ndiv} BRA.DIV, "
                  f"{len(local)} LDL/STL")
            if listing:
                for i in p[:-1]:
                    print(f"      {body[i][0]:#07x}  {body[i][1]}")


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    report(args[0] if args else os.path.join(ROOT, "cool-chic_b200", "csrc", "ccd_entropy.o"), "--list" in sys.argv)
