"""The stream-order contract on the host side (DESIGN.md §2, "Stream order"): every entry point that takes a stream, creates,
finalizes, loads or destroys a handle has a case in tests/test_gpu_stream_order.py, and fsn_api.cu never leaves a legacy-stream
zero-fill or a pageable copy unordered before a handle is used."""
import os
import re

import test_gpu_stream_order as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fsnplus_b200.h")
API = os.path.join(ROOT, "fullsubnet-plus_b200", "csrc", "fsn_api.cu")

# zero-fills and synchronous copies in functions that neither name a stream nor synchronise, each with the reason it is safe
ALLOW = {
    ("upload", "cudaMemcpy"): "called only by fsn_model_finalize, which synchronises the device before it returns",
}


def _decls():
    """(name, parameter text) of every function the header declares"""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return re.findall(r"\b(fsn_\w+)\s*\(([^;{]*?)\)\s*;", src)


def test_every_stream_entry_point_has_a_case():
    covered = {f for fns in G.CASES.values() for f in fns}
    need = sorted({n for n, p in _decls() if re.search(r"void\s*\*\s*stream\b", p) or re.search(r"_(create|finalize|load|destroy)$", n)})
    assert len(need) >= 40, need
    missing = [n for n in need if n not in covered]
    assert not missing, f"entry points without a stream-order case in test_gpu_stream_order.CASES: {missing}"
    for case in G.CASES:
        assert callable(getattr(G, case, None)), f"CASES names {case}, which test_gpu_stream_order does not define"


def _functions(src):
    """(name, body) of every top-level function definition: a signature that starts in column 0 (on one line or several) and ends
    with '{', to the next '}' in column 0"""
    out, name, body, sig = [], None, [], None
    for line in src.splitlines():
        if name is None:
            if sig is None:
                if re.match(r"^[A-Za-z]", line) and "(" in line and not line.startswith(
                        ("struct", "namespace", "static const struct", "#", "using", "typedef")) and not line.rstrip().endswith(";"):
                    sig = [line]
                else:
                    continue
            else:
                sig.append(line)
            text = " ".join(sig)
            if text.rstrip().endswith("{"):
                m = re.match(r"^.*?\b(\w+)\s*\(", text)
                name, body, sig = m.group(1), list(sig), None
            elif text.rstrip().endswith((";", "}")) or len(sig) > 8:
                sig = None
            continue
        body.append(line)
        if line.startswith("}"):
            out.append((name, "\n".join(body)))
            name = None
    return out


def _syncs_after(body, pos):
    """The function synchronises the device or a stream after offset pos"""
    return re.search(r"cudaDeviceSynchronize\(|cudaStreamSynchronize\(", body[pos:]) is not None


def _args(text, start):
    """The top-level arguments of the call whose '(' is at text[start]"""
    depth, cur, args = 0, "", []
    for ch in text[start:]:
        if ch == "(":
            depth += 1
            if depth == 1:
                continue
        elif ch == ")":
            depth -= 1
            if depth == 0:
                args.append(cur.strip())
                return args
        elif ch == "," and depth == 1:
            args.append(cur.strip())
            cur = ""
            continue
        cur += ch
    return args


def test_zero_fills_and_pageable_copies_are_ordered():
    """Every zero-filling ensure(..., true, ...) names a stream, or its function synchronises after it; every synchronous cudaMemcpy(
    is followed by a synchronise in its function (a pageable copy may return before its DMA lands, and the legacy stream does not
    order a non-blocking one)"""
    src = open(API).read()
    bad = []
    fns = _functions(src)
    # multi-line signatures included: every top-level '}' closes a function or a struct ('};')
    assert len(fns) == len(re.findall(r"(?m)^}(?!;)", src)), "a function definition the parser does not see"
    assert {"ensure_ws", "prepare", "step_slots", "run_audio", "fsn_model_forward_host", "fsn_chunk_stream_step"} <= {n for n, _ in fns}
    for name, body in fns:
        for m in re.finditer(r"\.ensure\(|->ensure\(", body):
            a = _args(body, m.end() - 1)
            if "true" not in a:
                continue
            i = a.index("true")
            stream = a[i + 1] if i + 1 < len(a) else "nullptr"
            if stream in ("nullptr", "0", "NULL") and not _syncs_after(body, m.end()) and (name, "ensure") not in ALLOW:
                bad.append(f"{name}: ensure({', '.join(a)}) zero-fills on the legacy stream and nothing synchronises after it")
        for m in re.finditer(r"\bcudaMemcpy\(", body):
            if not _syncs_after(body, m.end()) and (name, "cudaMemcpy") not in ALLOW:
                bad.append(f"{name}: cudaMemcpy( with no synchronise after it in the function")
    assert not bad, bad


def test_allow_list_is_live():
    """Every allow-list entry still names a function that has the call"""
    fns = dict(_functions(open(API).read()))
    for (name, call), why in ALLOW.items():
        assert why and name in fns and call + "(" in fns[name], (name, call)
    assert "cudaDeviceSynchronize()" in fns["fsn_model_finalize"]
