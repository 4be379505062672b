"""Where the C-ABI entries are defined, and the refusals and sizes of the entries defined outside api.cu, without a GPU.

An entry whose work no model code shares is defined in the file that implements it, inside that file's one
``extern "C"`` block, so the public header checks its signature and no forwarding function stands between them.  The
refusal table and the size grids pin the codes and byte counts those entries returned when they were still forwarded
from api.cu: every refused call returns before any CUDA call, so the fake device addresses are never dereferenced."""
import ctypes as C
import itertools
import json
import os
import re

import pytest

from sudo_rm_rf_b200 import _native as N

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "sudo_rm_rf_b200", "csrc")
HEADER = os.path.join(REPO, "include", "sudormrf_b200.h")
GOLDEN = os.path.join(REPO, "tests", "golden", "abi_size_queries.json")

BAD_CONFIG, BAD_ARGUMENT, WORKSPACE, UNSUPPORTED = -1, -2, -3, -5


# =====================================================================================================================
# 1. placement
# =====================================================================================================================
def _code(text):
    """The text without comments, preprocessor lines and string contents (except extern "C"'s), offsets kept."""
    def blank(m):
        s = m.group(0)
        if s == '"C"':
            return s
        if s[0] in "\"'":
            return s[0] + " " * (len(s) - 2) + s[-1]
        return re.sub(r"[^\n]", " ", s)
    text = re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', blank, text, flags=re.S)
    return re.sub(r"(?m)^[ \t]*#[^\n]*", lambda m: " " * len(m.group(0)), text)


def _close(code, i, open_, close):
    """The index just past the bracket that closes the one at code[i]."""
    depth = 0
    for j in range(i, len(code)):
        depth += {open_: 1, close: -1}.get(code[j], 0)
        if depth == 0:
            return j + 1
    raise AssertionError("unbalanced")


def _definitions(path):
    """[(name, in extern "C", body)] of every function defined at namespace scope of one source file."""
    code = _code(open(path).read())
    out, i, stack = [], 0, []          # stack: one entry per open brace: "extern", "ns" or a "body"
    while i < len(code):
        c = code[i]
        if c == "{":
            head = code[:i].rstrip()
            stack.append("extern" if head.endswith('extern "C"') else
                         "ns" if re.search(r"\bnamespace(\s+\w+)?$", head) else "body")
        elif c == "}":
            stack.pop()
        elif all(s != "body" for s in stack):
            m = re.compile(r"\b([A-Za-z_]\w*)\s*\(").match(code, i)
            if m and (i == 0 or not (code[i - 1].isalnum() or code[i - 1] == "_")):
                end = _close(code, m.end() - 1, "(", ")")
                rest = code[end:].lstrip()
                if rest.startswith("{"):
                    b0 = len(code) - len(rest)
                    b1 = _close(code, b0, "{", "}")
                    out.append((m.group(1), "extern" in stack, code[b0 + 1:b1 - 1]))
                    i = b1
                    continue
                i = end
                continue
        i += 1
    return out


def _forwards_only(body, callee):
    """True when the body is argument refusals (`if (...) return ...;`) and stream casts, then `return callee(...);`."""
    s = body.strip()
    while True:
        m = re.match(r"if\s*\(", s)
        if m:
            end = _close(s, m.end() - 1, "(", ")")
            r = re.match(r"\s*return\s[^;]*;", s[end:])
            if not r:
                return False
            s = s[end + r.end():].strip()
            continue
        m = re.match(r"(const\s+)?cudaStream_t\s+\w+\s*=\s*static_cast<cudaStream_t>\(\w+\);", s)
        if m:
            s = s[m.end():].strip()
            continue
        break
    m = re.match(r"return\s+" + callee + r"\s*\(", s)
    return bool(m) and s[_close(s, m.end() - 1, "(", ")"):].strip() == ";"


def _launcher_names():
    code = _code(open(os.path.join(CSRC, "launchers.cuh")).read())
    return re.findall(r"(?m)^(?:[\w:]+\s+)+\**(\w+)\(", code)


def test_launchers_are_the_ones_api_calls():
    """Every function launchers.cuh declares is called by api.cu, from a function that does more than forward."""
    names = _launcher_names()
    assert len(names) > 30
    defs = _definitions(os.path.join(CSRC, "api.cu"))
    unused = []
    for name in names:
        callers = [(f, body) for f, _, body in defs if re.search(r"\b" + name + r"\s*\(", body)]
        if not any(not (f.startswith("sdr_") and _forwards_only(body, name)) for f, body in callers):
            unused.append(name)
    assert not unused, f"declared for api.cu, which only forwards to them or never calls them: {unused}"


def test_every_entry_is_defined_once_inside_extern_c():
    declared = set(re.findall(r"\b(sdr_\w+)\s*\(", _code(open(HEADER).read())))
    assert declared == set(N.EXPORTED_SYMBOLS)
    found = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(".cu"):
            for name, in_extern, _ in _definitions(os.path.join(CSRC, f)):
                if name.startswith("sdr_"):
                    found.setdefault(name, []).append((f, in_extern))
    assert set(found) == declared, set(found) ^ declared
    for name, where in sorted(found.items()):
        assert len(where) == 1 and where[0][1], (name, where)


# =====================================================================================================================
# 2. refusals
# =====================================================================================================================
X = 1 << 20                       # a non-null device address aligned to 256 bytes
Y = 1 << 30                       # another one, far from X
M4, M8 = X + 4, X + 8             # misaligned for 8- and 16-byte buffers
BIG = 1 << 40


def ptrs(*v):
    """A host array of device pointers (the pyramids read it on the host)."""
    return (C.c_void_p * 8)(*(list(v) + [X] * (8 - len(v))))


# entry -> (parameter names in order, base arguments); each case changes one or two of them so that the call is
# refused
METRIC = dict(est=X, tgt=X, B=2, S=2, T=1000, stream=None)
ENTRIES = {
    "sdr_mixture_consistency": ("est mix out B S T wt scratch stream",
                                dict(METRIC, mix=X, out=X, wt=0, scratch=None)),
    "sdr_mixture_consistency_backward": ("est mix g ge gm B S T wt scratch stream",
                                         dict(METRIC, mix=X, g=X, ge=X, gm=None, wt=1, scratch=X)),
    "sdr_pairwise_neg_sdr": ("est tgt out B S T ty zm log scratch stream",
                             dict(METRIC, out=X, ty=1, zm=1, log=1, scratch=X)),
    "sdr_pairwise_neg_sdr_train": ("est tgt out coef B S T ty zm log scratch stream",
                                   dict(METRIC, out=X, coef=X, ty=1, zm=1, log=1, scratch=X)),
    "sdr_pairwise_neg_sdr_backward": ("est tgt coef g grad B S T stream", dict(METRIC, coef=X, g=X, grad=X)),
    "sdr_pit_sisdr": ("est tgt mix best perm B S T zm imp eps scratch stream",
                      dict(METRIC, mix=None, best=X, perm=X, zm=1, imp=0, eps=1e-8, scratch=X)),
    "sdr_stabilized_sisdr": ("est tgt best perm B rows ne na T zm imp eps scratch stream",
                             dict(METRIC, best=X, perm=X, rows=3, ne=3, na=2, zm=1, imp=0, eps=1e-8, scratch=X)),
    "sdr_snr_zero_refs": ("est tgt value perm coef B S T zm thr eps scratch stream",
                          dict(METRIC, value=X, perm=X, coef=X, zm=1, thr=-20.0, eps=1e-8, scratch=X)),
    "sdr_snr_zero_refs_backward": ("est tgt coef g grad B S T Tg stream", dict(METRIC, coef=X, g=X, grad=X, Tg=1000)),
    "sdr_bss_eval": ("ref est sdr sir sar perm B S T F cp scratch stream",
                     dict(METRIC, ref=X, sdr=X, sir=X, sar=X, perm=None, F=16, cp=1, scratch=X)),
    "sdr_bss_eval_mixture": ("ref est mix sdr sir sar perm msdr msir msar B S T F cp scratch stream",
                             dict(METRIC, ref=X, mix=X, sdr=X, sir=X, sar=X, perm=None, msdr=X, msir=X, msar=X, F=16,
                                  cp=1, scratch=X)),
    "sdr_stoi": ("ref est mix lengths out mout B S T fs scratch stream",
                 dict(METRIC, ref=X, mix=None, lengths=None, out=X, mout=None, T=30000, fs=16000, scratch=X)),
    "sdr_resample_poly": ("x out rows T up down scratch nb stream",
                          dict(x=X, out=Y, rows=2, T=1000, up=160, down=147, scratch=X, nb=BIG, stream=None)),
    "sdr_resample_stream_reset": ("state nb B rows C up down delay lead slots n stream",
                                  dict(state=X, nb=BIG, B=2, rows=1, C=441, up=8000, down=44100, delay=10, lead=0,
                                       slots=None, n=0, stream=None)),
    "sdr_resample_stream_step": ("state nb chunk zero out B rows C up down delay lead stream",
                                 dict(state=X, nb=BIG, chunk=Y, zero=None, out=Y, B=2, rows=1, C=441, up=8000,
                                      down=44100, delay=10, lead=0, stream=None)),
    "sdr_resample_stream_flush": ("state nb tail tl zero out B rows C up down delay lead stream",
                                  dict(state=X, nb=BIG, tail=Y, tl=100, zero=None, out=Y, B=2, rows=1, C=441,
                                       up=8000, down=44100, delay=10, lead=0, stream=None)),
    "sdr_window_gather": ("x batch B A T W H k0 M stream",
                          dict(x=X, batch=Y, B=2, A=1, T=100, W=10, H=5, k0=0, M=4, stream=None)),
    "sdr_window_merge": ("est carry perm out B S A T W H k0 M scratch stream",
                         dict(est=X, carry=X, perm=None, out=Y, B=2, S=2, A=1, T=100, W=10, H=5, k0=0, M=4,
                              scratch=X, stream=None)),
    "sdr_window_stream_reset": ("state B S A W H slots n stream",
                                dict(state=X, B=2, S=2, A=1, W=10, H=5, slots=None, n=0, stream=None)),
    "sdr_window_stream_reset_masked": ("state B S A W H mask stream",
                                       dict(state=X, B=2, S=2, A=1, W=10, H=5, mask=Y, stream=None)),
    "sdr_window_stream_gather": ("state chunk batch B S A C W H stream",
                                 dict(state=X, chunk=Y, batch=Y, B=2, S=2, A=1, C=20, W=10, H=5, stream=None)),
    "sdr_window_stream_merge": ("est state out B S A C W H scratch stream",
                                dict(est=Y, state=X, out=Y, B=2, S=2, A=1, C=20, W=10, H=5, scratch=X, stream=None)),
    "sdr_window_stream_flush": ("single est state out B S A W H scratch stream",
                                dict(single=Y, est=Y, state=X, out=Y, B=2, S=2, A=1, W=10, H=5, scratch=X,
                                     stream=None)),
    "sdr_depthwise_pyramid": ("y fin w5 bias gamma beta z stats0 scratch D samples C L stream",
                              dict(y=X, fin=None, w5=ptrs(), bias=ptrs(), gamma=ptrs(), beta=ptrs(), z=ptrs(),
                                   stats0=X, scratch=X, D=4, samples=2, C=8, L=128, stream=None)),
    "sdr_merge_pyramid": ("z scratch D m stats samples C L stream",
                          dict(z=ptrs(), scratch=X, D=4, m=X, stats=X, samples=2, C=8, L=128, stream=None)),
    "sdr_depthwise_pyramid_fused": ("y fin w5 bias gamma beta m stats0 stats_m scratch D samples C L stream",
                                    dict(y=X, fin=None, w5=ptrs(), bias=ptrs(), gamma=ptrs(), beta=ptrs(), m=Y,
                                         stats0=X, stats_m=X, scratch=X, D=4, samples=2, C=8, L=128, stream=None)),
}

SLOT_PAST_B = (C.c_int32 * 1)(2)

# (entry, case, overrides, code): single faults, then pairs, above all a misaligned buffer with a bad shape or rate
CASES = [
    ("sdr_mixture_consistency", "B=0", dict(B=0), BAD_ARGUMENT),
    ("sdr_mixture_consistency", "null est", dict(est=None), BAD_ARGUMENT),
    ("sdr_mixture_consistency", "weights 2", dict(wt=2), BAD_ARGUMENT),
    ("sdr_mixture_consistency", "weights 1, null scratch", dict(wt=1), BAD_ARGUMENT),
    ("sdr_mixture_consistency", "B S past int", dict(B=1 << 16, S=1 << 15), UNSUPPORTED),
    ("sdr_mixture_consistency", "B S past int, weights 2", dict(B=1 << 16, S=1 << 15, wt=2), UNSUPPORTED),
    ("sdr_mixture_consistency", "B S past int, null out", dict(B=1 << 16, S=1 << 15, out=None), BAD_ARGUMENT),

    ("sdr_mixture_consistency_backward", "misaligned scratch", dict(scratch=M8), BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "null scratch", dict(scratch=None), BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "null mix", dict(mix=None), BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "weights 2", dict(wt=2), BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "T=0", dict(T=0), BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "B S past int", dict(B=1 << 16, S=1 << 15), UNSUPPORTED),
    ("sdr_mixture_consistency_backward", "grid past int", dict(B=1 << 20, S=1 << 10, T=1 << 24), UNSUPPORTED),
    ("sdr_mixture_consistency_backward", "misaligned scratch, B S past int", dict(scratch=M8, B=1 << 16, S=1 << 15),
     BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "misaligned scratch, weights 0", dict(scratch=M8, wt=0), BAD_ARGUMENT),
    ("sdr_mixture_consistency_backward", "null est, B S past int", dict(est=None, B=1 << 16, S=1 << 15), BAD_ARGUMENT),

    ("sdr_pairwise_neg_sdr", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr", "null scratch", dict(scratch=None), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr", "type 3", dict(ty=3), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_pairwise_neg_sdr", "misaligned scratch, S=5", dict(scratch=M4, S=5), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr", "T=0, S=5", dict(T=0, S=5), BAD_ARGUMENT),

    ("sdr_pairwise_neg_sdr_train", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr_train", "misaligned coef", dict(coef=M4), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr_train", "null coef", dict(coef=None), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr_train", "S=0", dict(S=0), UNSUPPORTED),
    ("sdr_pairwise_neg_sdr_train", "misaligned coef, S=5", dict(coef=M4, S=5), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr_train", "misaligned scratch, S=5", dict(scratch=M4, S=5), BAD_ARGUMENT),

    ("sdr_pairwise_neg_sdr_backward", "misaligned coef", dict(coef=M4), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr_backward", "null grad", dict(grad=None), BAD_ARGUMENT),
    ("sdr_pairwise_neg_sdr_backward", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_pairwise_neg_sdr_backward", "misaligned coef, S=5", dict(coef=M4, S=5), BAD_ARGUMENT),

    ("sdr_pit_sisdr", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_pit_sisdr", "improvement without mixture", dict(imp=1), BAD_ARGUMENT),
    ("sdr_pit_sisdr", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_pit_sisdr", "misaligned scratch, S=5", dict(scratch=M4, S=5), BAD_ARGUMENT),
    ("sdr_pit_sisdr", "improvement without mixture, S=5", dict(imp=1, S=5), BAD_ARGUMENT),
    ("sdr_pit_sisdr", "null perm, S=5", dict(perm=None, S=5), BAD_ARGUMENT),

    ("sdr_stabilized_sisdr", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_stabilized_sisdr", "rows=0", dict(rows=0), BAD_ARGUMENT),
    ("sdr_stabilized_sisdr", "rows != n_est", dict(rows=2), BAD_ARGUMENT),
    ("sdr_stabilized_sisdr", "n_act > n_est", dict(na=4), UNSUPPORTED),
    ("sdr_stabilized_sisdr", "n_est=5", dict(ne=5, rows=5), UNSUPPORTED),
    ("sdr_stabilized_sisdr", "misaligned scratch, n_est=5", dict(scratch=M4, ne=5, rows=5), BAD_ARGUMENT),
    ("sdr_stabilized_sisdr", "rows != n_est, n_act > n_est", dict(rows=2, na=4), BAD_ARGUMENT),

    ("sdr_snr_zero_refs", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_snr_zero_refs", "misaligned coef", dict(coef=M4), BAD_ARGUMENT),
    ("sdr_snr_zero_refs", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_snr_zero_refs", "misaligned scratch, S=5", dict(scratch=M4, S=5), BAD_ARGUMENT),
    ("sdr_snr_zero_refs", "misaligned coef, S=5", dict(coef=M4, S=5), BAD_ARGUMENT),
    ("sdr_snr_zero_refs", "B=0, S=5", dict(B=0, S=5), BAD_ARGUMENT),

    ("sdr_snr_zero_refs_backward", "misaligned coef", dict(coef=M4), BAD_ARGUMENT),
    ("sdr_snr_zero_refs_backward", "Tg < T", dict(Tg=999), BAD_ARGUMENT),
    ("sdr_snr_zero_refs_backward", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_snr_zero_refs_backward", "misaligned coef, S=5", dict(coef=M4, S=5), BAD_ARGUMENT),
    ("sdr_snr_zero_refs_backward", "Tg < T, S=5", dict(Tg=999, S=5), BAD_ARGUMENT),

    ("sdr_bss_eval", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_bss_eval", "null sar", dict(sar=None), BAD_ARGUMENT),
    ("sdr_bss_eval", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_bss_eval", "F=0", dict(F=0), UNSUPPORTED),
    ("sdr_bss_eval", "S F past T", dict(T=10), UNSUPPORTED),
    ("sdr_bss_eval", "T=0", dict(T=0), BAD_ARGUMENT),
    ("sdr_bss_eval", "B (S + 1) past int", dict(B=1 << 30), UNSUPPORTED),
    ("sdr_bss_eval", "misaligned scratch, S=5", dict(scratch=M4, S=5), BAD_ARGUMENT),
    ("sdr_bss_eval", "misaligned scratch, B (S + 1) past int", dict(scratch=M4, B=1 << 30), BAD_ARGUMENT),

    ("sdr_bss_eval_mixture", "null mixture", dict(mix=None), BAD_ARGUMENT),
    ("sdr_bss_eval_mixture", "null mixture sar", dict(msar=None), BAD_ARGUMENT),
    ("sdr_bss_eval_mixture", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_bss_eval_mixture", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_bss_eval_mixture", "null mixture, S=5", dict(mix=None, S=5), BAD_ARGUMENT),
    ("sdr_bss_eval_mixture", "misaligned scratch, F past its limit", dict(scratch=M4, F=1 << 20), BAD_ARGUMENT),

    ("sdr_stoi", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_stoi", "mixture without its output", dict(mix=X), BAD_ARGUMENT),
    ("sdr_stoi", "rate 12345", dict(fs=12345), UNSUPPORTED),
    ("sdr_stoi", "B=0", dict(B=0), BAD_ARGUMENT),
    ("sdr_stoi", "misaligned scratch, rate 12345", dict(scratch=M4, fs=12345), BAD_ARGUMENT),
    ("sdr_stoi", "null scratch, rate 12345", dict(scratch=None, fs=12345), BAD_ARGUMENT),

    ("sdr_resample_poly", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_resample_poly", "up=0", dict(up=0), BAD_ARGUMENT),
    ("sdr_resample_poly", "ratio past 4096", dict(up=1, down=4097), UNSUPPORTED),
    ("sdr_resample_poly", "small scratch", dict(nb=8), WORKSPACE),
    ("sdr_resample_poly", "rows=0", dict(rows=0), BAD_ARGUMENT),
    ("sdr_resample_poly", "T past its limit", dict(T=(1 << 40) + 1), BAD_ARGUMENT),
    ("sdr_resample_poly", "misaligned scratch, ratio past 4096", dict(scratch=M4, up=1, down=4097), BAD_ARGUMENT),
    ("sdr_resample_poly", "ratio past 4096, small scratch", dict(up=1, down=4097, nb=8), UNSUPPORTED),
    ("sdr_resample_poly", "misaligned scratch, small scratch", dict(scratch=M4, nb=8), BAD_ARGUMENT),

    ("sdr_resample_stream_reset", "misaligned state", dict(state=M8), BAD_ARGUMENT),
    ("sdr_resample_stream_reset", "small state", dict(nb=8), WORKSPACE),
    ("sdr_resample_stream_reset", "slot past B", dict(slots=SLOT_PAST_B, n=1), BAD_ARGUMENT),
    ("sdr_resample_stream_reset", "misaligned state, equal rates", dict(state=M8, up=3, down=3), UNSUPPORTED),

    ("sdr_resample_stream_step", "null chunk", dict(chunk=None), BAD_ARGUMENT),
    ("sdr_resample_stream_step", "misaligned state", dict(state=M8), BAD_ARGUMENT),
    ("sdr_resample_stream_step", "small state", dict(nb=8), WORKSPACE),
    ("sdr_resample_stream_step", "equal rates", dict(up=2, down=2), UNSUPPORTED),
    ("sdr_resample_stream_step", "C not a multiple of q", dict(C=440), BAD_ARGUMENT),
    ("sdr_resample_stream_step", "misaligned state, small state", dict(state=M8, nb=8), WORKSPACE),
    ("sdr_resample_stream_step", "misaligned state, ratio past 4096", dict(state=M8, up=1, down=4097, C=4097),
     UNSUPPORTED),
    ("sdr_resample_stream_step", "null out, small state", dict(out=None, nb=8), BAD_ARGUMENT),

    ("sdr_resample_stream_flush", "negative tail", dict(tl=-1), BAD_ARGUMENT),
    ("sdr_resample_stream_flush", "null tail", dict(tail=None), BAD_ARGUMENT),
    ("sdr_resample_stream_flush", "misaligned state", dict(state=M8), BAD_ARGUMENT),
    ("sdr_resample_stream_flush", "small state", dict(nb=8), WORKSPACE),
    ("sdr_resample_stream_flush", "misaligned state, delay below its least", dict(state=M8, delay=9), BAD_ARGUMENT),
    ("sdr_resample_stream_flush", "null tail, small state", dict(tail=None, nb=8), BAD_ARGUMENT),

    ("sdr_window_gather", "null mixture", dict(x=None), BAD_ARGUMENT),
    ("sdr_window_gather", "H >= W", dict(H=10), BAD_ARGUMENT),
    ("sdr_window_gather", "past the last window", dict(k0=16), BAD_ARGUMENT),

    ("sdr_window_merge", "misaligned carry", dict(carry=M8), BAD_ARGUMENT),
    ("sdr_window_merge", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_window_merge", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_window_merge", "H < W/2", dict(H=4), BAD_ARGUMENT),
    ("sdr_window_merge", "misaligned carry, S=5", dict(carry=M8, S=5), BAD_ARGUMENT),
    ("sdr_window_merge", "misaligned scratch, S=5", dict(scratch=M4, S=5), BAD_ARGUMENT),
    ("sdr_window_merge", "S=5, past the last window", dict(S=5, k0=16), UNSUPPORTED),
    ("sdr_window_merge", "null output, S=5", dict(out=None, S=5), BAD_ARGUMENT),

    ("sdr_window_stream_reset", "misaligned state", dict(state=M8), BAD_ARGUMENT),
    ("sdr_window_stream_reset", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_window_stream_reset", "slot past B", dict(slots=SLOT_PAST_B, n=1), BAD_ARGUMENT),
    ("sdr_window_stream_reset_masked", "null mask", dict(mask=None), BAD_ARGUMENT),
    ("sdr_window_stream_reset_masked", "S=5, misaligned state", dict(S=5, state=M8), UNSUPPORTED),

    ("sdr_window_stream_gather", "null batch", dict(batch=None), BAD_ARGUMENT),
    ("sdr_window_stream_gather", "null chunk, C > 0", dict(chunk=None), BAD_ARGUMENT),
    ("sdr_window_stream_gather", "misaligned state", dict(state=M8), BAD_ARGUMENT),
    ("sdr_window_stream_gather", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_window_stream_gather", "C not a multiple of H", dict(C=21), BAD_ARGUMENT),
    ("sdr_window_stream_gather", "S=5, C not a multiple of H", dict(S=5, C=21), UNSUPPORTED),
    ("sdr_window_stream_gather", "misaligned state, C not a multiple of H", dict(state=M8, C=21), BAD_ARGUMENT),

    ("sdr_window_stream_merge", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_window_stream_merge", "misaligned state", dict(state=M8), BAD_ARGUMENT),
    ("sdr_window_stream_merge", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_window_stream_merge", "C not a multiple of H", dict(C=21), BAD_ARGUMENT),
    ("sdr_window_stream_merge", "S=5, misaligned scratch", dict(S=5, scratch=M4), UNSUPPORTED),
    ("sdr_window_stream_merge", "null scratch, S=5", dict(scratch=None, S=5), BAD_ARGUMENT),

    ("sdr_window_stream_flush", "misaligned scratch", dict(scratch=M4), BAD_ARGUMENT),
    ("sdr_window_stream_flush", "null estimates, W < 2H", dict(est=None, H=6), BAD_ARGUMENT),
    ("sdr_window_stream_flush", "S=5", dict(S=5), UNSUPPORTED),
    ("sdr_window_stream_flush", "S=5, misaligned scratch", dict(S=5, scratch=M4), UNSUPPORTED),
    ("sdr_window_stream_flush", "null single, S=5", dict(single=None, S=5), BAD_ARGUMENT),

    ("sdr_depthwise_pyramid", "null y", dict(y=None), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid", "null z", dict(z=None), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid", "null scratch", dict(scratch=None), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid", "null level weight", dict(w5=ptrs(X, X, None)), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid", "D=3", dict(D=3), UNSUPPORTED),
    ("sdr_depthwise_pyramid", "L=100", dict(L=100), UNSUPPORTED),
    ("sdr_depthwise_pyramid", "samples past the table", dict(samples=4097), UNSUPPORTED),
    ("sdr_depthwise_pyramid", "samples=0", dict(samples=0), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid", "misaligned y", dict(y=M4), UNSUPPORTED),
    ("sdr_depthwise_pyramid", "misaligned level", dict(z=ptrs(X, M8)), UNSUPPORTED),
    ("sdr_depthwise_pyramid", "null y, D=3", dict(y=None, D=3), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid", "misaligned y, null level weight", dict(y=M4, w5=ptrs(X, None)), BAD_ARGUMENT),

    ("sdr_merge_pyramid", "null z", dict(z=None), BAD_ARGUMENT),
    ("sdr_merge_pyramid", "null scratch", dict(scratch=None), BAD_ARGUMENT),
    ("sdr_merge_pyramid", "D=7", dict(D=7), UNSUPPORTED),
    ("sdr_merge_pyramid", "misaligned m", dict(m=M4), UNSUPPORTED),
    ("sdr_merge_pyramid", "misaligned level", dict(z=ptrs(X, X, X, M8)), UNSUPPORTED),
    ("sdr_merge_pyramid", "null m, D=7", dict(m=None, D=7), BAD_ARGUMENT),

    ("sdr_depthwise_pyramid_fused", "null m", dict(m=None), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid_fused", "null stats_m", dict(stats_m=None), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid_fused", "m overlaps y", dict(m=X + 16), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid_fused", "misaligned m", dict(m=Y + 4), UNSUPPORTED),
    ("sdr_depthwise_pyramid_fused", "D=7", dict(D=7), UNSUPPORTED),
    ("sdr_depthwise_pyramid_fused", "misaligned y", dict(y=M4), UNSUPPORTED),
    ("sdr_depthwise_pyramid_fused", "null stats_m, D=7", dict(stats_m=None, D=7), BAD_ARGUMENT),
    ("sdr_depthwise_pyramid_fused", "misaligned y, m overlaps y", dict(y=M4, m=X + 16), UNSUPPORTED),
]


@pytest.mark.parametrize("entry,kw,want", [(c[0], c[2], c[3]) for c in CASES], ids=[f"{c[0]}-{c[1]}" for c in CASES])
def test_refusal(entry, kw, want):
    names, base = ENTRIES[entry]
    a = dict(base, **kw)
    assert getattr(N.lib(), entry)(*[a[n] for n in names.split()]) == want


def test_every_moved_entry_has_refusals():
    assert {c[0] for c in CASES} == set(ENTRIES)


# =====================================================================================================================
# 3. size queries: every value over each grid, in itertools.product order, as recorded in tests/golden
# =====================================================================================================================
GRIDS = {
    "sdr_mixture_consistency_backward_scratch_bytes": ([0, 1, 3], [0, 1, 4], [0, 1, 1000, 1 << 20], [0, 1, 2]),
    "sdr_pairwise_neg_sdr_train_scratch_bytes": ([0, 2], [0, 1, 4, 5], [0, 1, 5000, 1 << 22]),
    "sdr_pairwise_neg_sdr_coef_bytes": ([0, 1, 7], [0, 1, 2, 4, 5]),
    "sdr_pit_sisdr_scratch_bytes": ([0, 1, 7], [0, 1, 2, 4, 5]),
    "sdr_stabilized_sisdr_scratch_bytes": ([0, 3], [0, 1, 2, 4, 5], [0, 1, 2, 4, 5]),
    "sdr_snr_zero_refs_scratch_bytes": ([0, 2], [0, 1, 4, 5], [0, 1, 5000, 1 << 22]),
    "sdr_snr_zero_refs_coef_bytes": ([0, 1, 7], [0, 1, 2, 4, 5]),
    "sdr_bss_eval_scratch_bytes": ([0, 2], [1, 2, 4, 5], [0, 10, 1000, 16000], [0, 1, 16, 512, 513]),
    "sdr_stoi_scratch_bytes": ([0, 2], [1, 3], [0, 100, 30000], [8000, 10000, 16000, 44100, 12345]),
    "sdr_resample_poly_scratch_bytes": ([0, 1, 2, 3, 160], [0, 1, 2, 3, 147, 4097]),
    "sdr_resample_stream_state_bytes": ([0, 2], [1, 2], [441, 440], [8000, 1], [44100, 2], [0, 10, 100], [0, 5]),
    "sdr_window_count": ([0, 1, 9, 10, 11, 100], [2, 10, 16], [1, 5, 8, 10]),
    "sdr_window_carry_bytes": ([0, 2], [1, 4, 5], [1, 2], [1, 2, 10, 1 << 24, (1 << 24) + 1]),
    "sdr_window_merge_scratch_bytes": ([0, 3], [0, 1, 4, 5], [0, 1, 7]),
    "sdr_window_stream_state_bytes": ([0, 2], [1, 4, 5], [1, 2], [10, 16000], [4, 5, 8000, 10]),
    "sdr_window_stream_merge_scratch_bytes": ([0, 2], [1, 5], [0, 10, 15], [0, 5]),
    "sdr_window_stream_flush_scratch_bytes": ([0, 2], [0, 1, 4, 5]),
    "sdr_window_stream_launch_count": ([0, 2], [2, 5], [1], [10, 21], [10], [5, 10]),
    "sdr_pyramid_scratch_bytes": ([0, 1, 4096, 4097], [8, 128], [3, 4, 5, 6, 7], [100, 128, 512, 4000]),
}


def test_size_queries():
    want = json.load(open(GOLDEN))
    assert set(want) == set(GRIDS)
    lib = N.lib()
    for entry, grid in GRIDS.items():
        got = [getattr(lib, entry)(*args) for args in itertools.product(*grid)]
        assert got == want[entry], entry
