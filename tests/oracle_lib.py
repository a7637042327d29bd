"""TEST INFRASTRUCTURE: ctypes access to oracle/liboracle.so (the CPU restatement), the unmodified
reference built into oracle/_ref (binaries + libfastga_ref.so) and the stored results of its runs."""
import contextlib
import ctypes as C
import hashlib
import json
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_SO = os.path.join(REF_DIR, "libfastga_ref.so")

_orc = None


def have_ref():
    return os.path.exists(os.path.join(REF_DIR, "FastGA")) and os.path.exists(REF_SO)


def orc():
    global _orc
    if _orc is None:
        if not os.path.exists(ORACLE_SO):
            subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-o", ORACLE_SO,
                                   os.path.join(ROOT, "oracle", "fastga_oracle.c")])
        _orc = C.CDLL(ORACLE_SO)
        _orc.orc_gix_build.restype = C.c_int64
        _orc.orc_merge.restype = C.c_int64
        _orc.orc_syncmers.restype = C.c_int64
        _orc.orc_new_work.restype = C.c_void_p
        if hasattr(_orc, "orc_search"):
            _orc.orc_search.restype = C.c_int64
    return _orc


class OrcSeed(C.Structure):
    _fields_ = [("plen", C.c_uint8), ("comp", C.c_uint8), ("icont", C.c_uint16), ("jcont", C.c_uint16),
                ("ipost", C.c_uint32), ("jpost", C.c_uint32)]


SEED_DT = np.dtype([("plen", "u1"), ("comp", "u1"), ("icont", "u2"), ("jcont", "u2"),
                    ("ipost", "u4"), ("jpost", "u4")], align=True)


class OrcLayout(C.Structure):
    _fields_ = [("anti_bits", C.c_int), ("band_bits", C.c_int), ("jc_bits", C.c_int), ("ic_bits", C.c_int),
                ("amxpos", C.c_int64), ("bmxpos", C.c_int64)]


def contig_rank(clen):
    """rank of each contig in the decreasing-length order; lengths must be pairwise distinct so
    the libc qsort tie order (GIXmake.c:1959) cannot matter"""
    clen = np.asarray(clen)
    perm = np.argsort(-clen, kind="stable").astype(np.int32)
    rank = np.empty_like(perm)
    rank[perm] = np.arange(len(clen), dtype=np.int32)
    return perm, rank


def gix_build(genome, crank):
    """oracle table of a formats.Genome: (n,2) uint64 records [lo,hi] + pstart"""
    o = orc()
    nc = genome.ncontig
    seqs = [np.ascontiguousarray(genome.contig(c)) for c in range(nc)]
    arr = (C.c_void_p * nc)(*[s.ctypes.data for s in seqs])
    tab = C.c_void_p()
    pstart = np.zeros((1 << 24) + 1, dtype=np.uint32)
    crank = np.ascontiguousarray(crank, dtype=np.int32)
    n = o.orc_gix_build(nc, arr, genome.clen.ctypes.data_as(C.c_void_p), crank.ctypes.data_as(C.c_void_p),
                        C.byref(tab), pstart.ctypes.data_as(C.c_void_p))
    out = np.ctypeslib.as_array(C.cast(tab, C.POINTER(C.c_uint64)), shape=(max(n, 1), 2))[:n].copy()
    o.orc_free(tab)
    return out, pstart


def merge(T1, T2, pstart2, freq=10):
    o = orc()
    T1 = np.ascontiguousarray(T1, dtype=np.uint64)
    T2 = np.ascontiguousarray(T2, dtype=np.uint64)
    sl = C.c_int64()
    args = [T1.ctypes.data_as(C.c_void_p), C.c_int64(len(T1)), T2.ctypes.data_as(C.c_void_p),
            C.c_int64(len(T2)), pstart2.ctypes.data_as(C.c_void_p), C.c_int(freq)]
    n = o.orc_merge(*args, None, C.byref(sl))
    seeds = np.zeros(n, dtype=SEED_DT)
    o.orc_merge(*args, seeds.ctypes.data_as(C.c_void_p), C.byref(sl))
    return seeds, sl.value


def self_merge(T, pstart, freq=10):
    """SELF mode (FastGA A): every entry of the one table against its own block (orc_self_merge)"""
    o = orc()
    T = np.ascontiguousarray(T, dtype=np.uint64)
    sl = C.c_int64()
    args = [T.ctypes.data_as(C.c_void_p), C.c_int64(len(T)), pstart.ctypes.data_as(C.c_void_p), C.c_int(freq)]
    o.orc_self_merge.restype = C.c_int64
    n = o.orc_self_merge(*args, None, C.byref(sl))
    seeds = np.zeros(n, dtype=SEED_DT)
    o.orc_self_merge(*args, seeds.ctypes.data_as(C.c_void_p), C.byref(sl))
    return seeds, sl.value


def seed_records(seeds, layout, sort=True):
    o = orc()
    out = np.zeros((len(seeds), 2), dtype=np.uint64)
    L = OrcLayout(*layout)
    o.orc_seed_records(seeds.ctypes.data_as(C.c_void_p), C.c_int64(len(seeds)), C.byref(L),
                       out.ctypes.data_as(C.c_void_p), C.c_int(1 if sort else 0))
    return out


# ------------------------------------------------------------------------------------------
#  the unmodified reference
# ------------------------------------------------------------------------------------------

#  What a test compared against the reference is stored in tests/golden/reference_runs.json, so the
#  comparison runs from a plain checkout.  With FGB_RECORD_REFERENCE=1 (and oracle/_ref built) every
#  reference() call recomputes its entry from the reference and rewrites the file.
GOLDEN_RUNS = os.path.join(ROOT, "tests", "golden", "reference_runs.json")
_golden = None


def digest(*parts):
    """md5 of the inputs of a reference run (arrays, lists of arrays, numbers, strings)"""
    h = hashlib.md5()
    def feed(x):
        if isinstance(x, (list, tuple)):
            h.update(b"[%d]" % len(x))
            for y in x:
                feed(y)
        elif isinstance(x, np.ndarray):
            h.update(str(x.dtype).encode() + str(x.shape).encode())
            h.update(np.ascontiguousarray(x).tobytes())
        else:
            h.update(repr(x).encode())
    feed(parts)
    return h.hexdigest()


def reference(key, inputs, compute):
    """The reference's result for `key` on `inputs` (a digest()): compute() -- which runs oracle/_ref
    and returns JSON data -- when recording, the stored result otherwise."""
    global _golden
    if _golden is None:
        with open(GOLDEN_RUNS) as f:
            _golden = json.load(f)
    if os.environ.get("FGB_RECORD_REFERENCE") == "1":
        if not have_ref():
            raise RuntimeError("FGB_RECORD_REFERENCE=1 needs oracle/_ref (build with FASTGA_REFERENCE set)")
        _golden[key] = {"inputs": inputs, "result": compute()}
        with open(GOLDEN_RUNS, "w") as f:          # one line per run
            f.write("{\n" + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(_golden[k], separators=(",", ":")))
                                       for k in sorted(_golden)) + "\n}\n")
    g = _golden[key]
    assert g["inputs"] == inputs, "%s: inputs changed since the reference run was recorded" % key
    return g["result"]


def ref_alignments(wd, a, b, threads=8, extra=()):
    """FastGA -v -k -T<n> -1:ref <extra> a [b] in workdir: -v counters + count and md5 of the canonical
    records (aln_md5), and md5 of the same lines in the file's order (aln_order_md5)"""
    st = parse_fastga_log(ref_fastga(wd, a, b, threads=threads, extra=extra))
    recs = oneview_records(os.path.join(wd, "ref.1aln"), ordered=True)
    st.update(records=len(recs), aln_md5=md5_lines(sorted(recs)), aln_order_md5=md5_lines(recs))
    return st


class Path(C.Structure):                     # align.h
    _fields_ = [("trace", C.c_void_p), ("tlen", C.c_int), ("diffs", C.c_int), ("abpos", C.c_int),
                ("bbpos", C.c_int), ("aepos", C.c_int), ("bepos", C.c_int)]


class Alignment(C.Structure):
    _fields_ = [("path", C.POINTER(Path)), ("flags", C.c_uint32), ("aseq", C.c_void_p), ("bseq", C.c_void_p),
                ("alen", C.c_int), ("blen", C.c_int)]


def path_key(abpos, bbpos, aepos, bepos, diffs, tlen, trace):
    """short digest of one Local_Alignment result: the path's ends, diffs and trace bytes"""
    h = np.array([abpos, bbpos, aepos, bepos, diffs, tlen], dtype=np.int32).tobytes()
    return hashlib.md5(h + np.asarray(trace).astype(np.uint8).tobytes()).hexdigest()[:12]


def ref_local_alignments(calls, freq, ave_corr=0.7):
    """path_key of the reference's Local_Alignment (libfastga_ref.so, New_Align_Spec(ave_corr, 100, freq))
    for every call (framed a, framed b, comp, low, hgh, anti, lbord, hbord)"""
    ref = C.CDLL(REF_SO)
    ref.New_Work_Data.restype = C.c_void_p
    ref.New_Align_Spec.restype = C.c_void_p
    ref.New_Align_Spec.argtypes = [C.c_double, C.c_int, C.POINTER(C.c_float), C.c_int]
    ref.Local_Alignment.argtypes = [C.POINTER(Alignment), C.c_void_p, C.c_void_p] + [C.c_int] * 5
    work = ref.New_Work_Data()
    spec = ref.New_Align_Spec(ave_corr, 100, (C.c_float * 4)(*[float(v) for v in freq]), 0)
    out = []
    for a, b, comp, low, hgh, anti, lb, hb in calls:
        p = Path()
        al = Alignment(C.pointer(p), 2 if comp else 0, a.ctypes.data + 1, b.ctypes.data + 1, len(a) - 2, len(b) - 2)
        assert ref.Local_Alignment(C.byref(al), work, spec, low, hgh, anti, lb, hb) == 0
        rt = np.ctypeslib.as_array(C.cast(p.trace, C.POINTER(C.c_uint16)), shape=(max(p.tlen, 1),))[:p.tlen]
        out.append(path_key(p.abpos, p.bbpos, p.aepos, p.bepos, p.diffs, p.tlen, rt))
    return out


def script_key(script, diffs):
    """short digest of one edit script (int entries as Compute_Trace_PTS leaves them) and its diffs"""
    return hashlib.md5(np.asarray(script, dtype=np.int32).tobytes() + b"%d" % diffs).hexdigest()[:12]


_ref_trace = None


def _ref_trace_lib():
    """libfastga_ref.so with its Error_Buffer pointed at a buffer, so that a record the reference rejects
    makes the call return 1 instead of exiting the process; plus one Work_Data for every call"""
    global _ref_trace
    if _ref_trace is None:
        ref = C.CDLL(REF_SO)
        buf = C.create_string_buffer(1 << 16)
        C.c_void_p.in_dll(ref, "Error_Buffer").value = C.addressof(buf)
        ref.New_Work_Data.restype = C.c_void_p
        ref.Compute_Trace_PTS.argtypes = [C.POINTER(Alignment), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        _ref_trace = (ref, buf, ref.New_Work_Data())
    return _ref_trace


def ref_trace_pts_raw(records, gA, gB):
    """Compute_Trace_PTS(aln, work, 100, GREEDIEST, 1, -1) on every record of `records` (fields (n, 9),
    toff and pool as lib.Alignments holds them) as ALNtoPAF.c:251-278 calls it: A and B in separate
    buffers (so the band is unbounded), strand-C records against the complement of their B contig.
    Per record (script, diffs), or None where the reference rejects the trace points."""
    ref, _, work = _ref_trace_lib()
    A, B, BC = {}, {}, {}
    out = []
    for i in range(len(records)):
        comp, ar, br, ab, bb, ae, be, df, tl = (int(x) for x in records.fields[i])
        if ar not in A:
            A[ar] = _framed(gA.contig(ar))
        if comp and br not in BC:
            BC[br] = _framed(3 - gB.contig(br)[::-1])
        elif not comp and br not in B:
            B[br] = _framed(gB.contig(br))
        pts = records.pool[int(records.toff[i]):int(records.toff[i]) + tl].astype(np.uint16)  # Decompress_TraceTo16
        p = Path(pts.ctypes.data, tl, df, ab, bb, ae, be)
        a, b = A[ar], (BC[br] if comp else B[br])
        al = Alignment(C.pointer(p), 2 if comp else 0, a.ctypes.data + 1, b.ctypes.data + 1, len(a) - 2, len(b) - 2)
        if ref.Compute_Trace_PTS(C.byref(al), work, 100, 0, 1, -1) != 0:
            out.append(None)
            continue
        sc = np.ctypeslib.as_array(C.cast(p.trace, C.POINTER(C.c_int32)), shape=(max(p.tlen, 1),))[:p.tlen].copy()
        out.append((sc, p.diffs))
    return out


def ref_trace_pts(records, gA, gB):
    """ref_trace_pts_raw as JSON data: per record script_key(script, diffs), or "fail" """
    return [("fail" if r is None else script_key(*r)) for r in ref_trace_pts_raw(records, gA, gB)]


def ref_env():
    env = dict(os.environ)
    env["PATH"] = REF_DIR + os.pathsep + env.get("PATH", "")
    return env


def run_ref(args, cwd, timeout=3600):
    r = subprocess.run(args, cwd=cwd, env=ref_env(), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=timeout)
    if r.returncode != 0:
        raise RuntimeError("reference command failed: %s\n%s" % (" ".join(args), r.stdout[-2000:]))
    return r.stdout


def ref_fastga(workdir, a, b, out="ref", threads=8, extra=()):
    """FastGA -v -k -T<n> -1:<out> a [b] in workdir (b None: SELF mode); returns the -v log"""
    return run_ref(["FastGA", "-v", "-k", "-T%d" % threads, "-P" + workdir, "-1:" + out] + list(extra) +
                   ([a, b] if b is not None else [a]), cwd=workdir)


def parse_fastga_log(log):
    log = log.replace("\r", "\n")
    d = {}
    m = re.search(r"Total seeds = ([\d,]+), ave\. len = ([\d.]+)", log)
    if m:
        d["seeds"] = int(m.group(1).replace(",", ""))
        d["avelen"] = float(m.group(2))
    m = re.search(r"Total hits over \d+bp = (\d+), (\d+) aln's, (\d+) non-redundant", log)
    if m:
        d["hits"], d["alns"], d["kept"] = int(m.group(1)), int(m.group(2)), int(m.group(3))
    return d


def oneview_records(path, ordered=False):
    """Canonical form of a .1aln: one text line per alignment ('A ..| R | D ..| T ..| X ..'),
    sorted (SURVEY 8c); ordered: in the file's order instead."""
    out = subprocess.run([os.path.join(REF_DIR, "ONEview"), path], stdout=subprocess.PIPE, text=True,
                         check=True).stdout
    recs, cur = [], None
    for line in out.split("\n"):
        if line.startswith("A "):
            if cur is not None:
                recs.append(cur)
            cur = line
        elif cur is not None and line[:2] in ("R", "R ", "D ", "T ", "X "):
            cur += " | " + line
        elif cur is not None and line.startswith("R"):
            cur += " | " + line
    if cur is not None:
        recs.append(cur)
    if not ordered:
        recs.sort()
    return recs


def md5_lines(lines):
    h = hashlib.md5()
    for l in lines:
        h.update(l.encode() + b"\n")
    return h.hexdigest()


def read_gdb_ascii(path):
    """contig lengths, scaffold names etc. of a .1gdb through ONEview"""
    out = subprocess.run([os.path.join(REF_DIR, "ONEview"), path], stdout=subprocess.PIPE, text=True,
                         check=True).stdout
    clen, names, scaf, sbeg = [], [], [], []
    pos = 0
    for line in out.split("\n"):
        if line.startswith("S "):
            names.append(line.split(" ", 2)[2])
            pos = 0
        elif line.startswith("G "):
            pos += int(line.split()[1])
        elif line.startswith("C "):
            n = int(line.split()[1])
            clen.append(n)
            scaf.append(len(names) - 1)
            sbeg.append(pos)
            pos += n
    return np.array(clen, np.int64), names, np.array(scaf, np.int32), np.array(sbeg, np.int64)


# ------------------------------------------------------------------------------------------
#  chain scan + extension through the oracle
# ------------------------------------------------------------------------------------------

class OrcSpec(C.Structure):
    _fields_ = [("tspace", C.c_int), ("path_ave", C.c_int), ("score", C.POINTER(C.c_int16)),
                ("table", C.POINTER(C.c_int16))]


class OrcParams(C.Structure):
    _fields_ = [("chain_break", C.c_int), ("chain_min", C.c_int), ("align_min", C.c_int),
                ("align_rate", C.c_double)]


OVL_DT = np.dtype([("comp", "i4"), ("aread", "i4"), ("bread", "i4"), ("abpos", "i4"), ("bbpos", "i4"),
                   ("aepos", "i4"), ("bepos", "i4"), ("diffs", "i4"), ("tlen", "i4"), ("grp", "i4"),
                   ("toff", "i8")], align=True)


def make_spec(freq, ave_corr=0.7, tspace=100):
    o = orc()
    tabs = np.zeros(65536, dtype=np.int16)
    ave = C.c_int()
    f = np.ascontiguousarray(freq, dtype=np.float32)
    o.orc_align_spec(C.c_double(ave_corr), f.ctypes.data_as(C.c_void_p), tabs.ctypes.data_as(C.c_void_p),
                     C.byref(ave))
    spec = OrcSpec(tspace, ave.value, C.cast(tabs.ctypes.data, C.POINTER(C.c_int16)),
                   C.cast(tabs.ctypes.data + 65536, C.POINTER(C.c_int16)))
    return spec, tabs, ave.value


def _framed(a):
    b = np.empty(len(a) + 2, dtype=np.int8)
    b[0] = 4
    b[-1] = 4
    b[1:-1] = a
    return b


CALL_DT = np.dtype([("comp", "i4"), ("ctg1", "i4"), ("ctg2", "i4"), ("low", "i4"), ("hgh", "i4"), ("anti", "i4"),
                    ("lbord", "i4"), ("hbord", "i4"), ("rec", "i4"), ("abpos", "i4"), ("bbpos", "i4"),
                    ("aepos", "i4"), ("bepos", "i4"), ("diffs", "i4"), ("tlen", "i4"), ("pass0", "i4"),
                    ("npass", "i4"), ("pad", "i4"), ("toff", "i8")])
PASS_DT = np.dtype([(n, "i4") for n in ("call", "s", "waves", "maxband", "narrowspan", "maxsnake", "aend", "bend",
                                        "stall", "endempty", "aspan", "da0", "da1", "db0", "db1", "maxhop")])


def search(recs, layout, gA, gB, perm1, perm2, freq, chain_break=2000, chain_min=170, align_min=100,
           align_rate=0.3):
    """oracle alignments in reference discovery order: (records, trace pool, nhit)"""
    return _search(recs, layout, gA, gB, perm1, perm2, freq, chain_break, chain_min, align_min, align_rate,
                   False)[:3]


def search_calls(recs, layout, gA, gB, perm1, perm2, freq, chain_break=2000, chain_min=170, align_min=100,
                 align_rate=0.3):
    """search(), and every Local_Alignment call it made, in discovery order: (records, trace pool, nhit,
    calls, passes).  calls: CALL_DT rows -- the call's arguments (original contig numbers), rec = 1 where
    it produced a record, its path (trace bytes "trace") and its passes [pass0, pass0+npass); passes:
    PASS_DT rows, what every wave pass went through (oracle/fastga_oracle.c orc_pass)."""
    return _search(recs, layout, gA, gB, perm1, perm2, freq, chain_break, chain_min, align_min, align_rate,
                   True)


def call_key(c):
    """path_key of one logged call (a CALL_DT row and its trace bytes)"""
    return path_key(c["abpos"], c["bbpos"], c["aepos"], c["bepos"], c["diffs"], c["tlen"], c["trace"])


def _search(recs, layout, gA, gB, perm1, perm2, freq, chain_break, chain_min, align_min, align_rate, logged):
    o = orc()
    spec, tabs, _ = make_spec(freq, 1.0 - align_rate)
    A = [_framed(gA.contig(c)) for c in range(gA.ncontig)]
    AC = [_framed(3 - gA.contig(c)[::-1]) for c in range(gA.ncontig)]
    B = [_framed(gB.contig(c)) for c in range(gB.ncontig)]
    pa = (C.c_void_p * gA.ncontig)(*[x.ctypes.data + 1 for x in A])
    pac = (C.c_void_p * gA.ncontig)(*[x.ctypes.data + 1 for x in AC])
    pb = (C.c_void_p * gB.ncontig)(*[x.ctypes.data + 1 for x in B])
    L = OrcLayout(*layout)
    P = OrcParams(chain_break, chain_min, align_min, align_rate)
    o.orc_new_result.restype = C.c_void_p
    R = C.c_void_p(o.orc_new_result())
    recs = np.ascontiguousarray(recs, dtype=np.uint64)
    p1 = np.ascontiguousarray(perm1, dtype=np.int32)
    p2 = np.ascontiguousarray(perm2, dtype=np.int32)
    args = [recs.ctypes.data_as(C.c_void_p), C.c_int64(len(recs)), C.byref(L), C.byref(P), C.byref(spec),
            p1.ctypes.data_as(C.c_void_p), p2.ctypes.data_as(C.c_void_p), pa, pac,
            gA.clen.ctypes.data_as(C.c_void_p), pb, gB.clen.ctypes.data_as(C.c_void_p), R]
    calls = passes = None
    if logged:
        for f in ("orc_new_calllog", "orc_calllog_call", "orc_calllog_pass", "orc_calllog_traces"):
            getattr(o, f).restype = C.c_void_p
        for f in ("orc_calllog_calls", "orc_calllog_passes", "orc_search_calls"):
            getattr(o, f).restype = C.c_int64
        for f in ("orc_calllog_calls", "orc_calllog_passes", "orc_calllog_call", "orc_calllog_pass",
                  "orc_calllog_traces", "orc_free_calllog"):
            getattr(o, f).argtypes = [C.c_void_p]
        G = C.c_void_p(o.orc_new_calllog())
        n = o.orc_search_calls(*args, G)
        nc, npas = o.orc_calllog_calls(G), o.orc_calllog_passes(G)

        def take(ptr, dt, count):
            if count == 0:
                return np.zeros(0, dtype=dt)
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(count * dt.itemsize,)).view(dt).copy()
        raw = take(o.orc_calllog_call(G), CALL_DT, nc)
        passes = take(o.orc_calllog_pass(G), PASS_DT, npas)
        tl = int((raw["toff"] + raw["tlen"]).max()) if nc else 0
        pool = take(o.orc_calllog_traces(G), np.dtype(np.uint8), tl)
        o.orc_free_calllog(G)
        calls = [dict({f: int(c[f]) for f in CALL_DT.names},
                      trace=pool[int(c["toff"]):int(c["toff"]) + int(c["tlen"])]) for c in raw]
    else:
        n = o.orc_search(*args)
    o.orc_result_ovls.restype = C.c_void_p
    o.orc_result_traces.restype = C.c_void_p
    o.orc_result_hits.restype = C.c_int64
    o.orc_result_ovls.argtypes = o.orc_result_traces.argtypes = o.orc_result_hits.argtypes = [C.c_void_p]
    nhit = o.orc_result_hits(R)
    if n > 0:
        ov = np.ctypeslib.as_array(C.cast(o.orc_result_ovls(R), C.POINTER(C.c_uint8)),
                                   shape=(n * OVL_DT.itemsize,)).view(OVL_DT).copy()
        tl = int((ov["toff"] + ov["tlen"]).max())
        tp = np.ctypeslib.as_array(C.cast(o.orc_result_traces(R), C.POINTER(C.c_uint8)), shape=(max(tl, 1),)).copy()
    else:
        ov = np.zeros(0, dtype=OVL_DT)
        tp = np.zeros(0, dtype=np.uint8)
    o.orc_free_result.argtypes = [C.c_void_p]
    o.orc_free_result(R)
    return ov, tp, nhit, calls, passes


CHAIN_TRIPLE_DT = np.dtype([("b", "i8"), ("m", "i8"), ("e", "i8"), ("isnew", "i8"), ("key", "i8"), ("cdiag", "i8"),
                            ("h0", "i8"), ("nh", "i8")])
CHAIN_HIT_DT = np.dtype([("alow", "i8"), ("ahgh", "i8"), ("dgmin", "i8"), ("dgmax", "i8"), ("nseed", "i8")])


def chains(recs, layout, chain_break=2000, chain_min=170):
    """the oracle's chain scan alone (orc_chains, the scan orc_search extends from): (triples, hits).
    triples: every scanned band-pair triple in scan order -- seeds [b, m) of band cdiag, [m, e) of band
    cdiag + 1, isnew, (strand, contig pair) key, its chains hits[h0 : h0 + nh]; hits: every chain that
    qualifies, in discovery order -- alow, ahgh, dgmin, dgmax as the scan holds them when it counts the
    hit (the coordinates of the device's ChainHit) and the number of seeds of the chain."""
    o = orc()
    o.orc_chains.restype = None
    recs = np.ascontiguousarray(recs, dtype=np.uint64)
    L = OrcLayout(*layout)
    counts = np.zeros(2, dtype=np.int64)
    args = [recs.ctypes.data_as(C.c_void_p), C.c_int64(len(recs)), C.byref(L), C.c_int(chain_break),
            C.c_int(chain_min)]
    o.orc_chains(*args, None, None, counts.ctypes.data_as(C.c_void_p))
    trip = np.zeros(int(counts[0]), dtype=CHAIN_TRIPLE_DT)
    hits = np.zeros(int(counts[1]), dtype=CHAIN_HIT_DT)
    o.orc_chains(*args, trip.ctypes.data_as(C.c_void_p), hits.ctypes.data_as(C.c_void_p),
                 counts.ctypes.data_as(C.c_void_p))
    return trip, hits


def pack_overlaps(ov, tp, rank1, rank2, jb, ib):
    """oracle alignments (discovery order) -> the packed record buffer the device stage emits, so the
    product's host filter can be run on them"""
    from fastga_b200 import lib
    parts = []
    for i, r in enumerate(ov):
        pk = (int(r["comp"]) << (jb + ib)) | (int(rank1[r["aread"]]) << jb) | int(rank2[r["bread"]])
        h = np.zeros(1, dtype=lib.RAW_HDR_DT)
        h["triple"], h["pairkey"] = i, pk
        for f in ("abpos", "bbpos", "aepos", "bepos", "diffs", "tlen"):
            h[f] = r[f]
        tr = bytes(tp[int(r["toff"]):int(r["toff"]) + int(r["tlen"])])
        tr += b"\0" * ((-len(tr)) % 8)
        parts.append(h.tobytes())
        parts.append(tr)
    buf = np.frombuffer(b"".join(parts), dtype=np.uint8) if parts else np.zeros(0, np.uint8)
    return lib.overlaps_from_buffer(buf)


FILTER_COUNTERS = ("s1_same_keep_o", "s1_same_drop_o", "s1_start_keep_o", "s1_start_drop_o", "s1_end_keep_o",
                   "s1_end_drop_o", "s2_b_disjoint", "s2_fuse", "s2_fuse_dead_o", "s2_fuse_w_owns",
                   "s2_box_drop_w", "s2_box_drop_o", "s2_apart_kept", "s2_cross", "s2_row_extended")


def filter(ov, tp, do_filter=True):
    """The oracle's redundancy filter and final order (orc_filter) on raw alignments ov (OVL_DT rows in
    discovery order; each run of equal ov["grp"] is one align_contigs call) with trace pool tp: the
    survivors in .1aln order, as a lib.Alignments"""
    from fastga_b200 import lib
    o = orc()
    o.orc_new_result.restype = C.c_void_p
    o.orc_filter.restype = C.c_int64
    o.orc_filter.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p]
    for f in ("orc_result_ovls", "orc_result_traces"):
        getattr(o, f).restype = C.c_void_p
        getattr(o, f).argtypes = [C.c_void_p]
    o.orc_free_result.argtypes = [C.c_void_p]
    ov = np.ascontiguousarray(ov, dtype=OVL_DT)
    tp = np.ascontiguousarray(tp, dtype=np.uint8)
    if tp.size == 0:
        tp = np.zeros(1, np.uint8)
    R = C.c_void_p(o.orc_new_result())
    n = o.orc_filter(ov.ctypes.data, len(ov), tp.ctypes.data, int(do_filter), R)
    if n > 0:
        out = np.ctypeslib.as_array(C.cast(o.orc_result_ovls(R), C.POINTER(C.c_uint8)),
                                    shape=(n * OVL_DT.itemsize,)).view(OVL_DT).copy()
        tl = int((out["toff"] + out["tlen"]).max())
        pool = np.ctypeslib.as_array(C.cast(o.orc_result_traces(R), C.POINTER(C.c_uint8)), shape=(max(tl, 1),)).copy()
    else:
        out, pool = np.zeros(0, dtype=OVL_DT), np.zeros(1, dtype=np.uint8)
    o.orc_free_result(R)
    fields = np.stack([out[f] for f in lib.ALN_FIELDS], axis=1).astype(np.int32).reshape(-1, 9)
    return lib.Alignments(fields, out["toff"].astype(np.int64), pool, len(ov))


def alignment_differences(got, want):
    """'' when two lib.Alignments hold the same records field by field and trace byte by trace byte, in
    the same order; else the first difference"""
    if len(got) != len(want):
        return "%d records != %d" % (len(got), len(want))
    for i in range(len(got)):
        if not np.array_equal(got.fields[i], want.fields[i]):
            return "record %d: %s != %s" % (i, got.fields[i].tolist(), want.fields[i].tolist())
        if not np.array_equal(got.trace(i), want.trace(i)):
            return "record %d: trace %s != %s" % (i, got.trace(i).tolist(), want.trace(i).tolist())
    return ""


def check_filters_and_order(r, st):
    """an oracle_pipeline(_self) result r against a ref_alignments run st: the product's filter on the
    oracle's raw records gave the oracle filter's records in its order, and that order is the
    reference's .1aln order"""
    d = alignment_differences(r["alns_product"], r["alns"])
    assert d == "", "fgb_filter != orc_filter: " + d
    assert md5_lines(r["order_lines"]) == st["aln_order_md5"]


def filter_counters():
    """per outcome (FILTER_COUNTERS), how often the last filter() went through each branch of the two
    sweeps; s2_fuse counts every fusion, s2_fuse_dead_o and s2_fuse_w_owns the fusions among them into
    an o its row had already eliminated and with a w that already owned a fused trace"""
    out = np.zeros(len(FILTER_COUNTERS), dtype=np.int64)
    orc().orc_filter_counters(out.ctypes.data_as(C.c_void_p))
    return dict(zip(FILTER_COUNTERS, (int(v) for v in out)))


def seed_layout(gA, gB):
    amx, bmx = int(gA.clen.max()), int(gB.clen.max())
    ab = int(amx + bmx).bit_length()
    return (ab, max(ab - 6, 1), int(max(gB.ncontig - 1, 1)).bit_length(),
            int(max(gA.ncontig - 1, 1)).bit_length(), amx, bmx)


def oracle_pipeline(gA, gB, rank=None, **kw):
    """The whole path through the CPU oracle, its own redundancy filter included.  Returns a dict; "alns"
    holds the oracle's final records, "alns_product" the product's host filter (fgb_filter) on the same
    raw records, "raw" the raw records and their trace pool.
    rank: (rank of every A contig, of every B contig) in place of contig_rank's, for genomes whose
    length ties leave the order open."""
    from fastga_b200 import lib
    pa, ra = contig_rank(gA.clen)
    pb, rb = contig_rank(gB.clen)
    if rank is not None:
        ra, rb = (np.asarray(r, dtype=np.int32) for r in rank)
        pa, pb = np.argsort(ra).astype(np.int32), np.argsort(rb).astype(np.int32)
    tA, sA = gix_build(gA, ra)
    tB, sB = gix_build(gB, rb)
    seeds, sumlen = merge(tA, tB, sB, kw.get("freq", 10))
    layout = seed_layout(gA, gB)
    recs = seed_records(seeds, layout)
    skw = {k: v for k, v in kw.items() if k in ("chain_break", "chain_min", "align_min", "align_rate")}
    ov, tp, nhit = search(recs, layout, gA, gB, pa, pb, gA.freq, **skw)
    ckw = {k: v for k, v in skw.items() if k in ("chain_break", "chain_min")}
    al = filter(ov, tp)
    fc = filter_counters()
    O = pack_overlaps(ov, tp, ra, rb, layout[2], layout[3])
    pal = lib.filter_overlaps(O.h, pa, pb, layout[2], layout[3])
    return dict(tabA=tA, tabB=tB, pstartA=sA, pstartB=sB, nseeds=len(seeds), sumlen=sumlen, seedrecs=recs,
                nhit=nhit, nchain=len(chains(recs, layout, **ckw)[1]), nraw=len(ov), alns=al,
                lines=al.canonical_lines(), order_lines=al.canonical_lines_unsorted(), alns_product=pal,
                filter_counters=fc, raw=(ov, tp), layout=layout, perm1=pa, perm2=pb, rank1=ra, rank2=rb)


SELF_COUNTERS = ("straddles", "stale_straddles", "lbord_calls", "hbord_calls")


@contextlib.contextmanager
def self_search(straddle_zero=False):
    """search() / search_calls() in SELF mode while inside: a contig against itself, forward strand, gets
    the band borders of align_contigs and no call across the main diagonal.  straddle_zero: such a
    straddle advances the tube with 0, as the CUDA path does, instead of the reference's stale bepos."""
    o = orc()
    o.orc_set_self(1)
    o.orc_set_straddle(int(straddle_zero))
    try:
        yield
    finally:
        o.orc_set_self(0)
        o.orc_set_straddle(0)


def self_counters():
    """what the last search went through in SELF mode (SELF_COUNTERS): straddles, straddles where the
    previous bepos lies past the chain's alow (so the two advances differ), calls with lbord >= 0 and
    calls with hbord >= 0"""
    out = np.zeros(4, dtype=np.int64)
    orc().orc_self_counters(out.ctypes.data_as(C.c_void_p))
    return dict(zip(SELF_COUNTERS, (int(v) for v in out)))


def oracle_pipeline_self(g, straddle_zero=False, **kw):
    """SELF mode (FastGA A) through the CPU oracle, its own redundancy filter included; "counters" holds
    self_counters() of the search, the rest as oracle_pipeline"""
    from fastga_b200 import lib
    pa, ra = contig_rank(g.clen)
    t, s = gix_build(g, ra)
    seeds, sumlen = self_merge(t, s, kw.get("freq", 10))
    layout = seed_layout(g, g)
    recs = seed_records(seeds, layout)
    skw = {k: v for k, v in kw.items() if k in ("chain_break", "chain_min", "align_min", "align_rate")}
    with self_search(straddle_zero):
        ov, tp, nhit = search(recs, layout, g, g, pa, pa, g.freq, **skw)
        cnt = self_counters()
    al = filter(ov, tp)
    fc = filter_counters()
    O = pack_overlaps(ov, tp, ra, ra, layout[2], layout[3])
    pal = lib.filter_overlaps(O.h, pa, pa, layout[2], layout[3])
    return dict(nseeds=len(seeds), sumlen=sumlen, nhit=nhit, nraw=len(ov), alns=al, lines=al.canonical_lines(),
                order_lines=al.canonical_lines_unsorted(), alns_product=pal, filter_counters=fc, raw=(ov, tp),
                counters=cnt, seedrecs=recs, layout=layout, perm=pa, rank=ra)
