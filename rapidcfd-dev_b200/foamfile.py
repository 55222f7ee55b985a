"""OpenFOAM on-disk formats for the hot path's inputs (SURVEY.md 8(f) rank 3): the
`constant/polyMesh/{points,faces,owner,neighbour,boundary}` files and `system/fvSolution`-style
dictionaries, so that real (also pre-decomposed `processorN/`) cases can drive the solver core
instead of the synthetic cubes of mesh.py.  Host-side set-up code; nothing here touches the GPU.

Restates (does not copy) the reference's readers:
 * dictionary syntax and look-up rules -- src/OpenFOAM/db/dictionary/dictionary.C:339-376 (exact
   keyword first, then the quoted regular-expression keys, most recently defined first
   :40-66,313-316), `$name` expansion (primitiveEntry.C), `//` and `/* */` comments;
 * `solution::solverDict` -- src/OpenFOAM/matrices/solution/solution.C:120 (`solvers` sub-dictionary);
 * list files -- FoamFile header + `N ( ... )`, ascii or binary (`format binary;`: raw int32 labels,
   float64 scalars/vectors; faces as the two lists of a faceCompactList);
 * geometry -- src/OpenFOAM/meshes/primitiveMesh/primitiveMeshFaceCentresAndAreas.C:78-138,
   primitiveMeshCellCentresAndVols.C:85-158; interpolation weights and delta coefficients --
   src/finiteVolume/interpolation/surfaceInterpolation/surfaceInterpolation/surfaceInterpolation.C:187-199,
   :271-366.
"""
import gzip
import os
import re
from dataclasses import dataclass, field

import numpy as np

# ---------------------------------------------------------------------------
# tokenizer + dictionary
# ---------------------------------------------------------------------------
_NUMBER = re.compile(r"[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)?")
_ENDS = set(" \t\r\n\f\v{}()[];\"")


def _strip_comments(text):
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    return re.sub(r"//[^\n]*", " ", text)


def tokenize(text):
    """Tokens as ISstream::read(token&) forms them (ISstream.C:140-420): punctuation, quoted strings, numbers, and words -- a word
    runs to the next white space, quote, `;`, `{`, `}` or bracket and may CONTAIN balanced parentheses (`div(phi,U)`,
    `div((nuEff*dev(T(grad(U)))))` are single keywords, ISstream::read(word&) :425-470); an unbalanced `)` ends it."""
    s = _strip_comments(text)
    out, i, n = [], 0, len(s)
    while i < n:
        c = s[i]
        if c.isspace():
            i += 1
        elif c == '"':
            j = i + 1
            while j < n and s[j] != '"':
                j += 2 if s[j] == "\\" else 1
            out.append(s[i:j + 1])
            i = j + 1
        elif c in "{}()[];":
            out.append(c)
            i += 1
        else:
            m = _NUMBER.match(s, i)
            if m and (m.end() == n or s[m.end()] in _ENDS):
                out.append(m.group())
                i = m.end()
                continue
            j, depth = i, 0
            while j < n:
                ch = s[j]
                if ch == "(":
                    depth += 1
                elif ch == ")":
                    if not depth:
                        break
                    depth -= 1
                elif ch.isspace() or ch in '{}[];"':
                    break
                j += 1
            out.append(s[i:j])
            i = j
    return out


_INT = re.compile(r"[-+]?\d+")
_FLOAT = re.compile(r"[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)?")


def _atom(tok):
    """word | number | quoted string (kept with its quotes removed, flagged by FoamString)"""
    if tok.startswith('"'):
        return FoamString(tok[1:-1])
    if _INT.fullmatch(tok):
        return int(tok)
    if _FLOAT.fullmatch(tok):      # digits required: `inf`, `nan`, `Infinity` stay words
        return float(tok)
    return tok


class FoamString(str):
    """a quoted token: as a dictionary key it is a regular expression (keyType::isPattern)"""


class FoamDict:
    """Ordered dictionary with OpenFOAM's look-up rules (dictionary.C:339-376)."""

    def __init__(self, parent=None, name=""):
        self.parent = parent
        self.name = name
        self.entries = {}       # keyword -> value, insertion ordered
        self.patterns = []      # (compiled regex, keyword), in definition order

    def add(self, key, value):
        if isinstance(key, FoamString):
            self.patterns.append((re.compile(str(key)), str(key)))
        self.entries[str(key)] = value

    def _find(self, key, recursive=False):
        if key in self.entries:
            return self.entries[key]
        for rx, kw in reversed(self.patterns):   # most recently defined pattern first
            if rx.fullmatch(key):
                return self.entries[kw]
        if recursive and self.parent is not None:
            return self.parent._find(key, True)
        raise KeyError(key)

    def found(self, key):
        try:
            self._find(key)
            return True
        except KeyError:
            return False

    def lookup(self, key, recursive=False):
        try:
            return self._find(key, recursive)
        except KeyError:
            raise KeyError(f"keyword {key} is undefined in dictionary \"{self.path()}\"") from None

    def lookupOrDefault(self, key, default):
        try:
            return self._find(key)
        except KeyError:
            return default

    def subDict(self, key):
        v = self.lookup(key)
        if not isinstance(v, FoamDict):
            raise KeyError(f"keyword {key} is not a sub-dictionary in \"{self.path()}\"")
        return v

    def path(self):
        return (self.parent.path() + "." if self.parent is not None and self.parent.name else "") + self.name

    def toc(self):
        return list(self.entries)

    def __contains__(self, key):
        return self.found(key)

    def __getitem__(self, key):
        return self.lookup(key)

    def to_python(self):
        return {k: (v.to_python() if isinstance(v, FoamDict) else v) for k, v in self.entries.items()}


class _Parser:
    def __init__(self, tokens):
        self.t = tokens
        self.i = 0

    def peek(self):
        return self.t[self.i] if self.i < len(self.t) else None

    def next(self):
        tok = self.peek()
        if tok is None:
            raise ValueError("unexpected end of dictionary")
        self.i += 1
        return tok

    def parse_dict_body(self, d, until=None):
        while True:
            tok = self.peek()
            if tok is None:
                if until is not None:
                    raise ValueError(f"missing '{until}' in dictionary {d.path()}")
                return d
            if tok == until:
                self.next()
                return d
            key = _atom(self.next())
            if isinstance(key, str) and not isinstance(key, FoamString) and key.startswith("#"):
                raise ValueError(f"directive {key} is not supported")
            if self.peek() == "{":
                self.next()
                sub = FoamDict(d, str(key))
                self.parse_dict_body(sub, "}")
                d.add(key, sub)
                continue
            vals = []
            while self.peek() != ";":
                if self.peek() is None:
                    raise ValueError(f"missing ';' after keyword {key} in {d.path()}")
                vals.append(self.parse_value(d))
            self.next()
            d.add(key, vals[0] if len(vals) == 1 else (None if not vals else vals))

    def parse_value(self, d):
        tok = self.next()
        if tok in ("(", "["):
            close = ")" if tok == "(" else "]"
            out = []
            while self.peek() != close:
                if self.peek() is None:
                    raise ValueError("unterminated list")
                if self.peek() == "{":       # list of dictionaries without keywords
                    self.next()
                    out.append(self.parse_dict_body(FoamDict(d), "}"))
                else:
                    out.append(self.parse_value(d))
            self.next()
            return out
        if tok == "{":
            return self.parse_dict_body(FoamDict(d), "}")
        a = _atom(tok)
        if isinstance(a, str) and not isinstance(a, FoamString) and a.startswith("$"):
            return d.lookup(a[1:], recursive=True)      # macro expansion, enclosing scopes included
        if isinstance(a, int) and self.peek() == "(":  # N ( ... ): sized list
            return self.parse_value(d)
        return a


def parse_dict(text, name=""):
    """Parse dictionary text (with or without a FoamFile header) into a FoamDict."""
    d = FoamDict(None, name)
    _Parser(tokenize(text)).parse_dict_body(d)
    return d


def read_dict(path):
    return parse_dict(_read_text(path), os.path.basename(path))


# ---------------------------------------------------------------------------
# fvSolution -> solver selection (lduMatrixSolver.C:43-140 reads exactly these keys)
# ---------------------------------------------------------------------------
_CONTROL_KEYS = {  # keyword -> (b200ldu_controls field, type)
    "tolerance": ("tolerance", float), "relTol": ("relTol", float), "maxIter": ("maxIter", int),
    "minIter": ("minIter", int), "nSweeps": ("nSweeps", int),
    "nCellsInCoarsestLevel": ("nCellsInCoarsestLevel", int), "mergeLevels": ("mergeLevels", int),
    "nPreSweeps": ("nPreSweeps", int), "preSweepsLevelMultiplier": ("preSweepsLevelMultiplier", int),
    "maxPreSweeps": ("maxPreSweeps", int), "nPostSweeps": ("nPostSweeps", int),
    "postSweepsLevelMultiplier": ("postSweepsLevelMultiplier", int), "maxPostSweeps": ("maxPostSweeps", int),
    "nFinestSweeps": ("nFinestSweeps", int), "interpolateCorrection": ("interpolateCorrection", "bool"),
    "scaleCorrection": ("scaleCorrection", "bool"), "directSolveCoarsest": ("directSolveCoarsest", "bool"),
}
_TRUE = {"yes", "on", "true", "y", "t", 1}
_FALSE = {"no", "off", "false", "n", "f", "none", 0}


def _switch(v):
    if v in _TRUE:
        return 1
    if v in _FALSE:
        return 0
    raise ValueError(f"bad Switch value {v!r}")


def solver_controls(fvSolution, fieldName):
    """(solver, preconditioner-or-smoother, controls) for `fieldName` from an fvSolution FoamDict.

    Mirrors solution::solverDict (solution.C) + lduMatrix::solver::New (lduMatrixSolver.C:43-140):
    `solver` selects the type; Krylov solvers read `preconditioner` (a word, or a dictionary whose
    `preconditioner` entry is the word -- lduMatrixPreconditioner.C:40-65), smoothSolver and GAMG
    read `smoother`.  `controls` holds only the keys present, named as in b200ldu_controls."""
    sd = fvSolution.subDict("solvers").subDict(fieldName)
    solver = sd.lookup("solver")
    second = ""
    if solver in ("PCG", "PBiCG", "PBiCGStab", "ICCG", "BICCG"):
        p = sd.lookupOrDefault("preconditioner", "DIC" if solver == "ICCG" else "DILU" if solver == "BICCG" else None)
        if p is None:
            raise KeyError(f"keyword preconditioner is undefined in dictionary \"{sd.path()}\"")
        second = p.lookup("preconditioner") if isinstance(p, FoamDict) else p
    elif solver in ("smoothSolver", "GAMG"):
        s = sd.lookup("smoother")
        second = s.lookup("smoother") if isinstance(s, FoamDict) else s
    controls = {}
    for key, (fld, typ) in _CONTROL_KEYS.items():
        if sd.found(key):
            v = sd.lookup(key)
            controls[fld] = _switch(v) if typ == "bool" else typ(v)
    return str(solver), str(second), controls


class FvSchemes:
    """system/fvSchemes as fvSchemes::read and the scheme look-ups interpret it (FV/finiteVolume/fvSchemes/fvSchemes.C:36-256,
    :425-580): per kind a sub-dictionary with an optional `default`; a look-up returns the entry for the name (exact keyword, then
    the quoted regular expressions, most recent first -- dictionary rules) and otherwise the default; `default none` means no
    default, and a name without an entry is then the reference's FatalIOError "keyword ... is undefined in dictionary".
    interpolationSchemes defaults to `linear` and snGradSchemes to `corrected` when the section is missing (:163-170, :207-214).
    Schemes come back as token lists, e.g. ["Gauss", "limitedLinear", 1]."""
    KINDS = ("ddtSchemes", "d2dt2Schemes", "interpolationSchemes", "divSchemes", "gradSchemes", "snGradSchemes", "laplacianSchemes")

    def __init__(self, d):
        self.sections, self.defaults = {}, {}
        for kind in self.KINDS:
            sec = d.subDict(kind) if d.found(kind) and isinstance(d.lookup(kind), FoamDict) else FoamDict(d, kind)
            if kind in ("ddtSchemes", "d2dt2Schemes") and not d.found(kind):
                sec.add("default", d.lookup("timeScheme") if d.found("timeScheme") else "none")   # the pre-1.6 keyword (:64-103)
            if kind == "interpolationSchemes" and not d.found(kind) and not sec.found("default"):
                sec.add("default", "linear")
            if kind == "snGradSchemes" and not d.found(kind) and not sec.found("default"):
                sec.add("default", "corrected")
            self.sections[kind] = sec
            dflt = self._tokens(sec.lookup("default")) if sec.found("default") else []
            self.defaults[kind] = [] if dflt[:1] == ["none"] else dflt
        self.flux = d.subDict("fluxRequired") if d.found("fluxRequired") else FoamDict(d, "fluxRequired")
        self.defaultFlux = False
        if self.flux.found("default") and self.flux.lookup("default") not in (None, "none"):
            self.defaultFlux = bool(_switch(self.flux.lookup("default")))

    @staticmethod
    def _tokens(v):
        return list(v) if isinstance(v, (list, tuple)) else [v]

    def _scheme(self, kind, name):
        sec, dflt = self.sections[kind], self.defaults[kind]
        if sec.found(name) or not dflt:
            if not sec.found(name):
                raise KeyError(f"keyword {name} is undefined in dictionary \"{sec.path()}\"")
            return self._tokens(sec.lookup(name))
        return list(dflt)

    def ddt(self, name):
        return self._scheme("ddtSchemes", name)

    def d2dt2(self, name):
        return self._scheme("d2dt2Schemes", name)

    def interpolation(self, name):
        return self._scheme("interpolationSchemes", name)

    def div(self, name):
        return self._scheme("divSchemes", name)

    def grad(self, name):
        return self._scheme("gradSchemes", name)

    def snGrad(self, name):
        return self._scheme("snGradSchemes", name)

    def laplacian(self, name):
        return self._scheme("laplacianSchemes", name)

    def fluxRequired(self, name):
        return True if self.flux.found(name) else self.defaultFlux


def convection_scheme(tokens):
    """`Gauss <interpolation scheme> [k]` of a divSchemes entry -> (scheme word for b200ldu_fv_limiter, k); `bounded Gauss ...` keeps
    the flag.  Unknown words answer like convectionScheme::New / surfaceInterpolationScheme::New: "Unknown ... scheme"."""
    t = list(tokens)
    bounded = t[:1] == ["bounded"]
    if bounded:
        t = t[1:]
    if t[:1] != ["Gauss"]:
        raise ValueError(f"Unknown convection type {t[0] if t else ''}\n\nValid convection types are :\n(Gauss bounded)")
    if len(t) < 2:
        raise ValueError("Discretisation scheme not specified")
    name = str(t[1])
    if name not in ("linear", "upwind", "limitedLinear", "vanLeer", "Minmod"):
        raise ValueError(f"Unknown discretisation scheme {name}\n\nValid schemes are :\n(Minmod limitedLinear linear upwind vanLeer)")
    k = float(t[2]) if name == "limitedLinear" and len(t) > 2 else 1.0
    return name, k, bounded


def alpha_controls(fvSolution, fvSchemes, fieldName="alpha.water"):
    """The controls of the interFoam phase-fraction step (rapidcfd-dev_b200/interfoam.py) from the `fieldName` solver entry of an
    fvSolution FoamDict and an FvSchemes, as FV/cfdTools/general/include/alphaControls.H, interfaceProperties.C:172-178 and MULES
    read them: nAlphaCorr, nAlphaSubCycles and cAlpha are required; MULESCorr and alphaApplyPrevCorr default to false, icAlpha to
    0; with MULESCorr, nLimiterIter is required (CMULESTemplates.C:95-98) and extremaCoeff defaults to 0 (:398-401) -- the explicit
    MULES::explicitSolve always sweeps three times (MULESTemplates.C:113).  alphaScheme / alpharScheme: (scheme word, k) of the
    divSchemes entries div(phi,alpha) / div(phirb,alpha); a scheme the limiter does not know is refused by name."""
    sd = fvSolution.subDict("solvers").subDict(fieldName)
    c = dict(nAlphaCorr=int(sd.lookup("nAlphaCorr")), nAlphaSubCycles=int(sd.lookup("nAlphaSubCycles")), cAlpha=float(sd.lookup("cAlpha")),
             MULESCorr=bool(_switch(sd.lookupOrDefault("MULESCorr", "no"))),
             alphaApplyPrevCorr=bool(_switch(sd.lookupOrDefault("alphaApplyPrevCorr", "no"))), icAlpha=float(sd.lookupOrDefault("icAlpha", 0)),
             nLimiterIter=3, extremaCoeff=float(sd.lookupOrDefault("extremaCoeff", 0.0)))
    if c["MULESCorr"]:
        c["nLimiterIter"] = int(sd.lookup("nLimiterIter"))
    for key, name in (("alphaScheme", "div(phi,alpha)"), ("alpharScheme", "div(phirb,alpha)")):
        c[key] = convection_scheme(fvSchemes.div(name))[:2]
    return c


# ---------------------------------------------------------------------------
# FoamFile list files
# ---------------------------------------------------------------------------
def _read_bytes(path):
    if not os.path.exists(path) and os.path.exists(path + ".gz"):
        path += ".gz"
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rb") as f:
        return f.read()


def _read_text(path):
    return _read_bytes(path).decode("latin-1")


_HEADER = re.compile(rb"FoamFile\s*\{(.*?)\}", re.S)


def _split_header(raw):
    """-> (header FoamDict, byte offset of the body)"""
    m = _HEADER.search(raw)
    if not m:
        return FoamDict(), 0
    return parse_dict(m.group(1).decode("latin-1")), m.end()


def _skip_ws_comments(raw, i):
    n = len(raw)
    while i < n:
        c = raw[i:i + 1]
        if c.isspace():
            i += 1
        elif raw[i:i + 2] == b"//":
            j = raw.find(b"\n", i)
            i = n if j < 0 else j + 1
        elif raw[i:i + 2] == b"/*":
            j = raw.find(b"*/", i)
            i = n if j < 0 else j + 2
        else:
            break
    return i


def _read_count(raw, i):
    i = _skip_ws_comments(raw, i)
    m = re.compile(rb"\d+").match(raw, i)
    if not m:
        raise ValueError("list size expected")
    return int(m.group()), m.end()


def _binary_block(raw, i, count, dtype):
    i = _skip_ws_comments(raw, i)
    if raw[i:i + 1] != b"(":
        raise ValueError("'(' expected before binary block")
    nbytes = count * np.dtype(dtype).itemsize
    a = np.frombuffer(raw, dtype=dtype, count=count, offset=i + 1).copy()
    j = i + 1 + nbytes
    if raw[j:j + 1] != b")":
        raise ValueError("')' expected after binary block")
    return a, j + 1


def read_list(path, kind):
    """kind: 'label' -> int32[N], 'scalar' -> float64[N], 'vector' -> float64[N,3],
    'face' -> (offsets int32[N+1], labels int32[...]) (CSR form of the faceList)."""
    raw = _read_bytes(path)
    hdr, i = _split_header(raw)
    binary = hdr.lookupOrDefault("format", "ascii") == "binary"
    n, i = _read_count(raw, i)
    if binary:
        if kind == "label":
            return _binary_block(raw, i, n, np.int32)[0]
        if kind == "scalar":
            return _binary_block(raw, i, n, np.float64)[0]
        if kind == "vector":
            return _binary_block(raw, i, 3 * n, np.float64)[0].reshape(n, 3)
        if kind == "face":   # faceCompactList: offsets (n entries = nFaces+1), then the labels
            offs, i = _binary_block(raw, i, n, np.int32)
            m, i = _read_count(raw, i)
            labels, _ = _binary_block(raw, i, m, np.int32)
            return offs, labels
        raise ValueError(kind)
    body = _strip_comments(raw[i:].decode("latin-1"))
    if kind == "label":
        a = np.array(re.findall(r"-?\d+", body), dtype=np.int64)
        return a[:n].astype(np.int32) if len(a) >= n else _short(path, n, len(a))
    if kind in ("scalar", "vector"):
        k = n * (3 if kind == "vector" else 1)
        a = np.array(re.findall(r"[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)?", body), dtype=np.float64)
        if len(a) < k:
            _short(path, k, len(a))
        return a[:k].reshape(n, 3) if kind == "vector" else a[:k]
    if kind == "face":
        offs = np.zeros(n + 1, dtype=np.int32)
        labels = []
        got = 0
        for m in re.finditer(r"(\d+)\s*\(([^()]*)\)", body):
            if got == n:
                break
            pts = m.group(2).split()
            if len(pts) != int(m.group(1)):
                raise ValueError(f"{path}: face {got} announces {m.group(1)} points, lists {len(pts)}")
            labels.extend(pts)
            offs[got + 1] = offs[got] + len(pts)
            got += 1
        if got < n:
            _short(path, n, got)
        return offs, np.array(labels, dtype=np.int32)
    raise ValueError(kind)


def _short(path, want, got):
    raise ValueError(f"{path}: expected {want} entries, found {got}")


_BANNER = """/*--------------------------------*- C++ -*----------------------------------*\\
| b200ldu foamfile.py                                                         |
\\*---------------------------------------------------------------------------*/
"""


def _header(cls, obj, binary, note=""):
    return (_BANNER + "FoamFile\n{\n    version     2.0;\n    format      %s;\n    class       %s;\n%s"
            "    location    \"constant/polyMesh\";\n    object      %s;\n}\n\n"
            % ("binary" if binary else "ascii", cls, note, obj)).encode()


def write_list(path, kind, data, binary=False, note=""):
    cls = {"label": "labelList", "scalar": "scalarField", "vector": "vectorField", "face": "faceList"}[kind]
    if kind == "face" and binary:
        cls = "faceCompactList"
    out = [_header(cls, os.path.basename(path), binary, note)]
    if kind == "face":
        offs, labels = data
        n = len(offs) - 1
        if binary:
            out += [b"%d\n(" % (n + 1), np.asarray(offs, np.int32).tobytes(), b")\n\n%d\n(" % len(labels),
                    np.asarray(labels, np.int32).tobytes(), b")\n"]
        else:
            lines = ["%d(%s)" % (offs[f + 1] - offs[f], " ".join(map(str, labels[offs[f]:offs[f + 1]])))
                     for f in range(n)]
            out.append(("%d\n(\n%s\n)\n" % (n, "\n".join(lines))).encode())
    else:
        a = np.asarray(data)
        n = len(a)
        if binary:
            raw = a.astype(np.int32 if kind == "label" else np.float64).tobytes()
            out += [b"%d\n(" % n, raw, b")\n"]
        elif kind == "vector":
            out.append(("%d\n(\n%s\n)\n" % (n, "\n".join("(%r %r %r)" % tuple(map(float, v)) for v in a))).encode())
        else:
            fmt = "%d" if kind == "label" else "%r"
            out.append(("%d\n(\n%s\n)\n" % (n, "\n".join(fmt % (int(v) if kind == "label" else float(v))
                                                          for v in a))).encode())
    with open(path, "wb") as f:
        f.write(b"".join(out))


# ---------------------------------------------------------------------------
# polyMesh
# ---------------------------------------------------------------------------
@dataclass
class PolyPatch:
    name: str
    type: str
    nFaces: int
    startFace: int
    myProcNo: int = -1
    neighbProcNo: int = -1
    neighbourPatch: str = ""


@dataclass
class PolyMesh:
    """owner/neighbour addressing (+ optional geometry) of one (sub-)domain."""
    owner: np.ndarray                 # int32 [nFaces] all faces
    neighbour: np.ndarray             # int32 [nInternalFaces]
    patches: list = field(default_factory=list)
    points: np.ndarray = None         # float64 [nPoints, 3]
    faceOffsets: np.ndarray = None
    faceLabels: np.ndarray = None

    @property
    def nInternalFaces(self):
        return len(self.neighbour)

    @property
    def nCells(self):
        return int(max(self.owner.max(), self.neighbour.max() if len(self.neighbour) else -1)) + 1

    # ---- LDU addressing as the C ABI takes it (lduAddressing: lower = owner of internal faces) ----
    def ldu(self):
        nI = self.nInternalFaces
        return self.owner[:nI].astype(np.int32), self.neighbour.astype(np.int32)

    def coupled_patches(self):
        return [p for p in self.patches if p.type in ("processor", "processorCyclic", "cyclic")]

    def coupled_interface_arrays(self):
        """(patchStart, faceCells, neighbRank) for b200ldu_addr_create: processor patches carry the
        neighbour rank, cyclic patches -(partner index + 1) among the coupled patches."""
        cps = self.coupled_patches()
        if not cps:
            return None, None, None
        index = {p.name: i for i, p in enumerate(cps)}
        start = np.zeros(len(cps) + 1, dtype=np.int32)
        cells, ranks = [], []
        for i, p in enumerate(cps):
            start[i + 1] = start[i] + p.nFaces
            cells.append(self.owner[p.startFace:p.startFace + p.nFaces])
            if p.type == "cyclic":
                if p.neighbourPatch not in index:
                    raise ValueError(f"cyclic patch {p.name}: neighbourPatch {p.neighbourPatch!r} not found")
                ranks.append(-(index[p.neighbourPatch] + 1))
            else:
                ranks.append(p.neighbProcNo)
        return start, np.concatenate(cells).astype(np.int32), np.array(ranks, dtype=np.int32)

    def boundary_face_cells(self):
        """faceCells of ALL boundary faces in patch order (fvPatch::faceCells)."""
        return self.owner[self.nInternalFaces:].astype(np.int32)

    # ---- geometry (needs points + faces) ----
    def face_centres_and_areas(self):
        """primitiveMeshFaceCentresAndAreas.C:78-138 (triangles direct, else triangle fan about the
        point average)."""
        p, offs, lab = self.points, self.faceOffsets, self.faceLabels
        nF = len(offs) - 1
        size = np.diff(offs)
        fid = np.repeat(np.arange(nF), size)
        cur = p[lab]
        nxt_idx = np.arange(len(lab)) + 1
        last = offs[1:] - 1
        nxt_idx[last] = offs[:-1]
        nxt = p[lab[nxt_idx]]
        fCentre = np.zeros((nF, 3))
        np.add.at(fCentre, fid, cur)
        fCentre /= size[:, None]
        fc = fCentre[fid]
        c = cur + nxt + fc
        nvec = np.cross(nxt - cur, fc - cur)
        a = np.linalg.norm(nvec, axis=1)
        sumN = np.zeros((nF, 3))
        sumA = np.zeros(nF)
        sumAc = np.zeros((nF, 3))
        np.add.at(sumN, fid, nvec)
        np.add.at(sumA, fid, a)
        np.add.at(sumAc, fid, a[:, None] * c)
        small = sumA < 1.0e-150  # ROOTVSMALL
        safe = np.where(small, 1.0, sumA)
        ctrs = np.where(small[:, None], fCentre, sumAc / safe[:, None] / 3.0)
        areas = np.where(small[:, None], 0.0, 0.5 * sumN)
        tri = np.nonzero(size == 3)[0]
        if len(tri):
            p0, p1, p2 = p[lab[offs[tri]]], p[lab[offs[tri] + 1]], p[lab[offs[tri] + 2]]
            ctrs[tri] = (p0 + p1 + p2) / 3.0
            areas[tri] = 0.5 * np.cross(p1 - p0, p2 - p0)
        return ctrs, areas

    def cell_centres_and_volumes(self, fCtrs=None, fAreas=None):
        """primitiveMeshCellCentresAndVols.C:85-158 (pyramids about the face-centre average)."""
        if fCtrs is None:
            fCtrs, fAreas = self.face_centres_and_areas()
        own, nei, nC, nI = self.owner, self.neighbour, self.nCells, self.nInternalFaces
        cEst = np.zeros((nC, 3))
        cnt = np.zeros(nC)
        np.add.at(cEst, own, fCtrs)
        np.add.at(cnt, own, 1)
        np.add.at(cEst, nei, fCtrs[:nI])
        np.add.at(cnt, nei, 1)
        cEst /= cnt[:, None]
        ctr = np.zeros((nC, 3))
        vol = np.zeros(nC)
        pyr = np.einsum("ij,ij->i", fAreas, fCtrs - cEst[own])
        np.add.at(ctr, own, pyr[:, None] * (0.75 * fCtrs + 0.25 * cEst[own]))
        np.add.at(vol, own, pyr)
        pyrN = np.einsum("ij,ij->i", fAreas[:nI], cEst[nei] - fCtrs[:nI])
        np.add.at(ctr, nei, pyrN[:, None] * (0.75 * fCtrs[:nI] + 0.25 * cEst[nei]))
        np.add.at(vol, nei, pyrN)
        ok = np.abs(vol) > 1e-300
        ctr = np.where(ok[:, None], ctr / np.where(ok, vol, 1.0)[:, None], cEst)
        return ctr, vol / 3.0

    def fv_geometry(self):
        """What the face-sum kernels and the coefficient builders consume: C, V, Sf, magSf (all faces),
        weights and deltaCoeffs of the internal faces (surfaceInterpolation.C:187-199, :300-312)."""
        Cf, Sf = self.face_centres_and_areas()
        C, V = self.cell_centres_and_volumes(Cf, Sf)
        nI = self.nInternalFaces
        own, nei = self.owner[:nI], self.neighbour
        SfdOwn = np.abs(np.einsum("ij,ij->i", Sf[:nI], Cf[:nI] - C[own]))
        SfdNei = np.abs(np.einsum("ij,ij->i", Sf[:nI], C[nei] - Cf[:nI]))
        w = SfdNei / (SfdOwn + SfdNei)
        delta = 1.0 / np.linalg.norm(C[nei] - C[own], axis=1)
        return dict(C=C, V=V, Cf=Cf, Sf=Sf, magSf=np.linalg.norm(Sf, axis=1), weights=w, deltaCoeffs=delta)

    def near_wall_dist(self, wallPatches=None):
        """nearWallDist::correct (finiteVolume/fvMesh/wallDist/nearWallDist.C:40-100): for every face of a wall patch, the
        distance from its cell centre to the nearest of the face and its point neighbours on the same patch
        (cellDistFuncs::getPointNeighbours / smallestDist, meshTools/cellDist/cellDistFuncs.C:82-170), each face taken as the
        triangle fan about its point average (face::nearestPoint).  Returns y of every boundary face in patch order, 0 on the
        other patches.  wallPatches: names of the wall patches (default: the patches of type wall).  Once per mesh."""
        C, _ = self.cell_centres_and_volumes()
        nI = self.nInternalFaces
        y = np.zeros(len(self.owner) - nI)
        for p in self.patches:
            if not (p.name in wallPatches if wallPatches is not None else p.type == "wall"):
                continue
            faces = [self.faceLabels[self.faceOffsets[f]:self.faceOffsets[f + 1]] for f in range(p.startFace, p.startFace + p.nFaces)]
            pointFaces = {}
            for i, f in enumerate(faces):
                for q in f:
                    pointFaces.setdefault(int(q), []).append(i)
            for i, f in enumerate(faces):
                nbrs = {i}.union(*(pointFaces[int(q)] for q in f))
                c = C[self.owner[p.startFace + i]]
                y[p.startFace - nI + i] = min(_face_distance(c, self.points[faces[j]]) for j in nbrs)
        return y


def _triangle_distance(p, a, b, c):
    """distance from p to the closest point of triangle abc (Ericson, Real-Time Collision Detection 5.1.5)"""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = ab @ ap, ac @ ap
    if d1 <= 0 and d2 <= 0:
        return float(np.linalg.norm(ap))
    bp = p - b
    d3, d4 = ab @ bp, ac @ bp
    if d3 >= 0 and d4 <= d3:
        return float(np.linalg.norm(bp))
    vc = d1 * d4 - d3 * d2
    if vc <= 0 and d1 >= 0 and d3 <= 0:
        return float(np.linalg.norm(p - (a + ab * (d1 / (d1 - d3)))))
    cp = p - c
    d5, d6 = ab @ cp, ac @ cp
    if d6 >= 0 and d5 <= d6:
        return float(np.linalg.norm(cp))
    vb = d5 * d2 - d1 * d6
    if vb <= 0 and d2 >= 0 and d6 <= 0:
        return float(np.linalg.norm(p - (a + ac * (d2 / (d2 - d6)))))
    va = d3 * d6 - d5 * d4
    if va <= 0 and (d4 - d3) >= 0 and (d5 - d6) >= 0:
        return float(np.linalg.norm(p - (b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6))))))
    den = 1.0 / (va + vb + vc)
    return float(np.linalg.norm(p - (a + ab * (vb * den) + ac * (vc * den))))


def _face_distance(p, pts):
    """distance from p to a face given by its points: the triangle itself, or the fan of triangles about the point average"""
    if len(pts) == 3:
        return _triangle_distance(p, pts[0], pts[1], pts[2])
    ctr = pts.mean(axis=0)
    return min(_triangle_distance(p, pts[k], pts[(k + 1) % len(pts)], ctr) for k in range(len(pts)))

def read_boundary(path):
    raw = _read_bytes(path)
    _, i = _split_header(raw)
    toks = tokenize(raw[i:].decode("latin-1"))
    if not toks:
        return []
    k = 0
    n = int(toks[k])
    k += 1
    if toks[k] != "(":
        raise ValueError(f"{path}: '(' expected")
    pr = _Parser(toks)
    pr.i = k + 1
    out = []
    for _ in range(n):
        name = pr.next()
        if pr.next() != "{":
            raise ValueError(f"{path}: '{{' expected after patch name {name}")
        d = pr.parse_dict_body(FoamDict(None, name), "}")
        out.append(PolyPatch(name, str(d.lookup("type")), int(d.lookup("nFaces")), int(d.lookup("startFace")),
                             int(d.lookupOrDefault("myProcNo", -1)), int(d.lookupOrDefault("neighbProcNo", -1)),
                             str(d.lookupOrDefault("neighbourPatch", ""))))
    return out


def read_poly_mesh(polyMeshDir, geometry=True):
    """Read constant/polyMesh (of a case or of a processorN directory)."""
    j = lambda f: os.path.join(polyMeshDir, f)
    owner = read_list(j("owner"), "label")
    neighbour = read_list(j("neighbour"), "label")
    pm = PolyMesh(owner, neighbour, read_boundary(j("boundary")))
    if len(neighbour) > len(owner):
        raise ValueError("neighbour list longer than owner list")
    nB = sum(p.nFaces for p in pm.patches)
    if pm.patches and pm.patches[0].startFace != len(neighbour):
        raise ValueError("first patch does not start at nInternalFaces")
    if len(neighbour) + nB != len(owner):
        raise ValueError("owner size != internal + boundary faces")
    lo, up = pm.ldu()
    if len(lo) and not (np.all(lo < up) and np.all(np.diff(lo) >= 0)):
        raise ValueError("internal faces are not in upper-triangular order (owner < neighbour, sorted by owner)")
    if geometry and (os.path.exists(j("points")) or os.path.exists(j("points.gz"))):
        pm.points = read_list(j("points"), "vector")
        pm.faceOffsets, pm.faceLabels = read_list(j("faces"), "face")
        if len(pm.faceOffsets) - 1 != len(owner):
            raise ValueError("faces and owner disagree on the number of faces")
    return pm


def write_poly_mesh(polyMeshDir, pm, binary=False):
    os.makedirs(polyMeshDir, exist_ok=True)
    j = lambda f: os.path.join(polyMeshDir, f)
    note = "    note        \"nPoints:%d  nCells:%d  nFaces:%d  nInternalFaces:%d\";\n" % (
        0 if pm.points is None else len(pm.points), pm.nCells, len(pm.owner), pm.nInternalFaces)
    write_list(j("owner"), "label", pm.owner, binary, note)
    write_list(j("neighbour"), "label", pm.neighbour, binary, note)
    if pm.points is not None:
        write_list(j("points"), "vector", pm.points, binary)
        write_list(j("faces"), "face", (pm.faceOffsets, pm.faceLabels), binary)
    body = ["%d\n(" % len(pm.patches)]
    for p in pm.patches:
        extra = ""
        if p.type in ("processor", "processorCyclic"):
            extra = "        myProcNo        %d;\n        neighbProcNo    %d;\n" % (p.myProcNo, p.neighbProcNo)
        if p.type == "cyclic":
            extra = "        neighbourPatch  %s;\n" % p.neighbourPatch
        body.append("    %s\n    {\n        type            %s;\n%s        nFaces          %d;\n"
                    "        startFace       %d;\n    }" % (p.name, p.type, extra, p.nFaces, p.startFace))
    body.append(")\n")
    with open(j("boundary"), "wb") as f:
        f.write(_header("polyBoundaryMesh", "boundary", False) + "\n".join(body).encode())


def from_hex_mesh(hm, rank=-1):
    """PolyMesh (with points and faces) of a mesh.HexMesh brick: the file set blockMesh /
    decomposePar would write for it (`rank` = myProcNo of a decomposed brick).  Boundary faces
    follow in patch order."""
    nx, ny, nz, h = hm.nx, hm.ny, hm.nz, hm.h
    i0, j0, k0 = hm.origin
    pid = lambda i, j, k: i + (nx + 1) * (j + (ny + 1) * k)
    ii, jj, kk = np.meshgrid(np.arange(nx + 1), np.arange(ny + 1), np.arange(nz + 1), indexing="ij")
    pts = np.zeros(((nx + 1) * (ny + 1) * (nz + 1), 3))
    pts[pid(ii, jj, kk).ravel()] = np.stack([(ii + i0) * h, (jj + j0) * h, (kk + k0) * h], axis=-1).reshape(-1, 3)

    def quad(c, axis, hi):
        """the 4 points of the face of cell c on side `hi` of `axis`, ordered so that the normal
        points along +axis for hi=1 and -axis for hi=0 (outward)."""
        i, j, k = c % nx, (c // nx) % ny, c // (nx * ny)
        o = [i, j, k]
        o[axis] = o[axis] + hi
        a, b = [(1, 2), (2, 0), (0, 1)][axis]   # right-handed pair: e_a x e_b = e_axis
        corners = []
        for da, db in ((0, 0), (1, 0), (1, 1), (0, 1)):
            q = list(o)
            q[a] = q[a] + da
            q[b] = q[b] + db
            corners.append(pid(q[0], q[1], q[2]))
        q4 = np.stack(corners, axis=-1)
        return q4 if hi else q4[..., ::-1]

    faces = [quad(hm.lower[hm.faceDir == d].astype(np.int64), d, 1) for d in range(3)]
    # internal faces must keep the mesh's own order: rebuild per face
    q_int = np.zeros((hm.nFaces, 4), dtype=np.int64)
    for d in range(3):
        q_int[hm.faceDir == d] = faces[d]
    owner = [hm.lower.astype(np.int32)]
    quads = [q_int]
    patches = []
    start = hm.nFaces
    for p in hm.patches:
        axis = int(np.argmax(np.abs(p.Sf[0]))) if len(p.Sf) else 0
        hi = 1 if (len(p.Sf) and p.Sf[0][axis] > 0) else 0
        quads.append(quad(p.faceCells.astype(np.int64), axis, hi))
        owner.append(p.faceCells.astype(np.int32))
        if p.kind == "processor":
            patches.append(PolyPatch(p.name, "processor", len(p.faceCells), start, rank, p.neighbRank))
        else:
            patches.append(PolyPatch(p.name, "wall", len(p.faceCells), start))
        start += len(p.faceCells)
    allq = np.concatenate(quads)
    offs = (4 * np.arange(len(allq) + 1)).astype(np.int32)
    return PolyMesh(np.concatenate(owner), hm.upper.astype(np.int32), patches, pts, offs,
                    allq.reshape(-1).astype(np.int32))


# ---------------------------------------------------------------------------
# decomposition (what decomposePar writes into processorN/constant/polyMesh)
# ---------------------------------------------------------------------------
def decompose_poly_mesh(pm, cellToProc):
    """Split `pm` by the cell -> rank map, following domainDecomposition's ordering
    (applications/utilities/parallelProcessing/decomposePar in OpenFOAM; not part of the reference
    tree, its conventions are what processorLduInterface relies on):
      * local cells and points keep their global relative order;
      * internal faces = global internal faces with both cells on the rank, in global order (upper-
        triangular order is preserved);
      * then the physical patches in their order (faces in global order, empty patches kept);
      * then one processor patch per neighbour rank in ascending rank order, its faces in global face
        order on BOTH sides (so face i of procBoundaryAtoB is face i of procBoundaryBtoA); the face is
        stored flipped where the local cell is the global neighbour.
    A cyclic face stays in its cyclic patch on the rank that owns its cell; processorCyclic patches (a
    cyclic pair split across ranks) are not produced -- keep both halves of a pair on one rank.
    Returns a list of (PolyMesh, cellGlobal, faceGlobal) per rank; faceGlobal < 0 marks a flipped face
    (-(f+1))."""
    cellToProc = np.asarray(cellToProc, dtype=np.int64)
    nP = int(cellToProc.max()) + 1 if len(cellToProc) else 1
    nI = pm.nInternalFaces
    own, nei = pm.owner.astype(np.int64), pm.neighbour.astype(np.int64)
    po, pn = cellToProc[own[:nI]], cellToProc[nei]
    out = []
    for r in range(nP):
        cells = np.nonzero(cellToProc == r)[0]
        local = -np.ones(pm.nCells, dtype=np.int64)
        local[cells] = np.arange(len(cells))
        f_int = np.nonzero((po == r) & (pn == r))[0]
        owner = [local[own[f_int]]]
        neigh = local[nei[f_int]]
        faceG = [f_int]
        patches = []
        start = len(f_int)
        for p in pm.patches:                                   # physical (and cyclic) patches
            if p.type in ("processor", "processorCyclic"):
                continue
            f = np.arange(p.startFace, p.startFace + p.nFaces)
            f = f[cellToProc[own[f]] == r]
            patches.append(PolyPatch(p.name, p.type, len(f), start, neighbourPatch=p.neighbourPatch))
            owner.append(local[own[f]])
            faceG.append(f)
            start += len(f)
        cut = np.nonzero(((po == r) | (pn == r)) & (po != pn))[0]   # internal faces cut by the decomposition
        other = np.where(po[cut] == r, pn[cut], po[cut])
        for nb in np.unique(other):
            f = cut[other == nb]                                  # global face order
            mine_is_owner = po[f] == r
            owner.append(local[np.where(mine_is_owner, own[f], nei[f])])
            faceG.append(np.where(mine_is_owner, f, -(f + 1)))
            patches.append(PolyPatch(f"procBoundary{r}to{int(nb)}", "processor", len(f), start, r, int(nb)))
            start += len(f)
        faceG = np.concatenate(faceG)
        sub = PolyMesh(np.concatenate(owner).astype(np.int32), neigh.astype(np.int32), patches)
        if pm.points is not None:
            gf = np.where(faceG >= 0, faceG, -faceG - 1)
            sizes = (pm.faceOffsets[gf + 1] - pm.faceOffsets[gf]).astype(np.int64)
            offs = np.zeros(len(gf) + 1, dtype=np.int64)
            np.cumsum(sizes, out=offs[1:])
            labels = np.empty(int(offs[-1]), dtype=np.int64)
            for i, (g, fl) in enumerate(zip(gf, faceG < 0)):
                pts = pm.faceLabels[pm.faceOffsets[g]:pm.faceOffsets[g + 1]]
                # a flipped face keeps its first point and reverses the rest (face::reverseFace)
                labels[offs[i]:offs[i + 1]] = pts if not fl else np.concatenate([pts[:1], pts[:0:-1]])
            used = np.unique(labels)
            pl = -np.ones(len(pm.points), dtype=np.int64)
            pl[used] = np.arange(len(used))
            sub.points = pm.points[used]
            sub.faceOffsets = offs.astype(np.int32)
            sub.faceLabels = pl[labels].astype(np.int32)
        out.append((sub, cells, faceG))
    return out


# ---------------------------------------------------------------------------
# field files (0/p, 0/U, ...: volScalarField / volVectorField / surfaceScalarField)
# ---------------------------------------------------------------------------
_FIELD_ENTRY = re.compile(rb"(internalField|value)\s+(uniform|nonuniform)\s+")


def read_field(path, nInternal=None):
    """Read a FoamFile field: dict(cls, dimensions, internalField, boundaryField={patch: dict(type, value?, ...)}).
    `uniform` values stay scalars / 3-vectors unless `nInternal` is given (then they are expanded);
    `nonuniform List<scalar|vector>` is read in ascii or binary (`format binary;` in the header)."""
    raw = _read_bytes(path)
    hdr, i0 = _split_header(raw)
    binary = hdr.lookupOrDefault("format", "ascii") == "binary"
    cls = str(hdr.lookupOrDefault("class", ""))

    def take_value(i):
        """parse `uniform X;` or `nonuniform List<T> N(...);` starting at i; returns (value, end offset)"""
        i = _skip_ws_comments(raw, i)
        if raw.startswith(b"uniform", i):
            j = raw.index(b";", i)
            toks = tokenize(raw[i + 7:j].decode("latin-1"))
            vals = [float(t) for t in toks if t not in ("(", ")")]
            return (np.array(vals) if len(vals) > 1 else vals[0]), j + 1
        if not raw.startswith(b"nonuniform", i):
            raise ValueError(f"{path}: uniform/nonuniform expected")
        i = _skip_ws_comments(raw, i + 10)
        m = re.compile(rb"List<(\w+)>").match(raw, i)
        if not m:
            raise ValueError(f"{path}: List<...> expected")
        kind = m.group(1).decode()
        ncmp = {"scalar": 1, "vector": 3, "symmTensor": 6, "tensor": 9}[kind]
        n, i = _read_count(raw, m.end())
        if binary:
            a, i = _binary_block(raw, i, n * ncmp, np.float64)
        else:
            i = _skip_ws_comments(raw, i)
            depth, j = 0, i
            while True:                       # matching ')' of the list
                c = raw[j:j + 1]
                if c == b"(":
                    depth += 1
                elif c == b")":
                    depth -= 1
                    if depth == 0:
                        break
                elif not c:
                    raise ValueError(f"{path}: unterminated list")
                j += 1
            a = np.array(re.findall(r"[-+]?(?:\d+\.?\d*|\.\d+)(?:[eE][-+]?\d+)?", raw[i:j + 1].decode("latin-1")),
                         dtype=np.float64)
            if len(a) != n * ncmp:
                _short(path, n * ncmp, len(a))
            i = j + 1
        i = raw.index(b";", i) + 1
        return (a.reshape(n, ncmp) if ncmp > 1 else a), i

    # cut the (possibly binary) values out, parse the rest as a dictionary
    values, pieces, pos = [], [], i0
    for m in _FIELD_ENTRY.finditer(raw, i0):
        if m.start() < pos:
            continue
        v, end = take_value(m.start(2))
        pieces.append(raw[pos:m.start(2)])
        pieces.append(b"__value%d__;" % len(values))
        values.append(v)
        pos = end
    pieces.append(raw[pos:])
    d = parse_dict(b"".join(pieces).decode("latin-1"))

    def resolve(x):
        if isinstance(x, str) and x.startswith("__value") and x.endswith("__"):
            return values[int(x[7:-2])]
        return x
    internal = resolve(d.lookup("internalField"))
    if nInternal is not None and (np.isscalar(internal) or np.ndim(internal) == 1 and cls.startswith("volVector")):
        internal = np.tile(np.atleast_1d(internal), (nInternal, 1)) if np.ndim(internal) == 1 else np.full(nInternal, internal)
    bf = {}
    for name, sub in d.subDict("boundaryField").entries.items():
        bf[name] = {k: resolve(v) for k, v in sub.entries.items()}
    return dict(cls=cls, dimensions=d.lookupOrDefault("dimensions", None), internalField=internal, boundaryField=bf)


def write_field(path, cls, dimensions, internalField, boundaryField, binary=False, location="0"):
    """Write a field file (the inverse of read_field for scalar / vector fields)."""
    def fmt_value(v):
        a = np.asarray(v, dtype=np.float64)
        if a.ndim == 0:
            return b"uniform %r" % float(a)
        if a.ndim == 1 and cls.startswith(("volVector", "surfaceVector")) and a.shape == (3,):
            return b"uniform (%r %r %r)" % tuple(map(float, a))
        kind = b"vector" if a.ndim == 2 else b"scalar"
        n = len(a)
        if binary:
            return b"nonuniform List<%s> %d(" % (kind, n) + a.tobytes() + b")"
        if a.ndim == 2:
            body = b"\n".join(b"(%r %r %r)" % tuple(map(float, r)) for r in a)
        else:
            body = b"\n".join(b"%r" % float(x) for x in a)
        return b"nonuniform List<%s> %d\n(\n" % (kind, n) + body + b"\n)"
    out = [_BANNER.encode(), ("FoamFile\n{\n    version     2.0;\n    format      %s;\n    class       %s;\n"
                              "    location    \"%s\";\n    object      %s;\n}\n\n"
                              % ("binary" if binary else "ascii", cls, location, os.path.basename(path))).encode(),
           ("dimensions      [%s];\n\n" % " ".join(str(x) for x in dimensions)).encode(),
           b"internalField   ", fmt_value(internalField), b";\n\nboundaryField\n{\n"]
    for name, entries in boundaryField.items():
        out.append(("    %s\n    {\n" % name).encode())
        for k, v in entries.items():
            if k == "value" or isinstance(v, (np.ndarray, float)):
                out += [("        %-15s " % k).encode(), fmt_value(v), b";\n"]
            else:
                out.append(("        %-15s %s;\n" % (k, v)).encode())
        out.append(b"    }\n")
    out.append(b"}\n")
    with open(path, "wb") as f:
        f.write(b"".join(out))
