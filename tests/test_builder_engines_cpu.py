"""The builder's exact parity list (SEQUENTIAL in test_builder_engines_gpu) reaches every distance engine, and each
side of every bound that picks an engine's layout.  The engine choice is read from the sources, so a new engine or a
moved bound fails here until the list covers it:

- DistDispatch (granne_b200.cu): the engine of each element kind, and the f32 chunk counts (dim / 32) that have a
  DistF32<FULL> of their own; every other f32 width takes DistF32Generic.
- engine_tiles (granne_b200.cu): DistF32Generic stages rows of up to `d.full <= 64` chunks and loads wider ones
  directly.
- stage_dense (granne_b200.cu) pads i8 rows to 32 bytes, and DistI8::load_query (search_kernels.cuh) splits a row into
  16-byte chunks and uses sub-warp groups for up to `chunks <= 32u` of them, one candidate at a time above that.
- DistSum::dists (search_kernels.cuh) sums a row in passes of 128 floats."""
import os
import re

from test_builder_engines_gpu import SEQUENTIAL

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "granne_b200", "csrc")
KINDS = {"kAngularI8": "angular_int", "kSumEmbeddings": "embeddings"}  # the element kinds with one engine each


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _one(pattern, text, what):
    found = re.findall(pattern, text)
    assert len(found) == 1, "%s: %r matches %d times" % (what, pattern, len(found))
    return found[0]


def _block(text, start):
    """From `start` to the first line that closes a top-level struct or function."""
    i = text.index(start)
    return text[i:text.index("\n}", i)]


def engine_choice():
    cu, kernels = _source("granne_b200.cu"), _source("search_kernels.cuh")
    dispatch = _block(cu, "struct DistDispatch {")
    by_kind = {KINDS[k]: e for k, e in re.findall(r"case gb::(\w+): return f\(Engine<gb::(\w+)>\{\}\);", dispatch)}
    fixed = {}
    for label, full in re.findall(r"case (\d+): return f\(Engine<gb::DistF32<(\d+)>>\{\}\);", dispatch):
        assert label == full, "case %s dispatches DistF32<%s>" % (label, full)
        fixed[int(full)] = "DistF32<%s>" % full
    generic = _one(r"default: return f\(Engine<gb::(\w+)>\{\}\);", dispatch, "DistDispatch default")
    named = set(re.findall(r"Engine<gb::(\w+(?:<\d+>)?)>", dispatch))
    assert named == set(by_kind.values()) | set(fixed.values()) | {generic}, named
    staged_max = int(_one(r"fixed_chunks < 0 && d\.full <= (\d+)\)", _block(cu, "EngineTiles engine_tiles("),
                          "engine_tiles"))
    pad = int(_one(r"d\.row_stride = \(dim \+ (\d+)u\) & ~\d+u;\s*// rows start on 32-byte", cu, "i8 row stride")) + 1
    load_query = _block(kernels, "struct DistI8 {")
    chunk_bytes = int(_one(r"chunks = ix\.row_stride / (\d+)u;", load_query, "DistI8 chunks"))
    sub_warp_max = int(_one(r"C = chunks <= (\d+)u \? chunks : 0u;", load_query, "DistI8::load_query"))
    sum_pass = int(_one(r"for \(int i0 = 0; i0 < dim; i0 \+= (\d+)\)", _block(kernels, "struct DistSum {"),
                        "DistSum pass"))

    def engine(kind, dim):
        """(engine, layout) that serves `kind` rows of `dim`."""
        if kind in by_kind:
            e = by_kind[kind]
            if e == "DistI8":
                chunks = -(-dim // pad) * pad // chunk_bytes
                return e, "sub-warp groups" if chunks <= sub_warp_max else "one row at a time"
            return e, "one pass" if dim <= sum_pass else "several passes"
        full = dim // 32
        if full in fixed:
            return fixed[full], "tail" if dim % 32 else "no tail"
        return generic, "staged" if full <= staged_max else "direct"

    return engine, set(by_kind.values()) | set(fixed.values()) | {generic}


def test_each_builder_case_reaches_the_engine_it_names():
    engine, _ = engine_choice()
    for kind, dim, _, _, named in SEQUENTIAL:
        assert engine(kind, dim) == named, (kind, dim)


def test_the_builder_parity_list_reaches_every_engine():
    engine, engines = engine_choice()
    reached = {engine(kind, dim) for kind, dim, _, _, _ in SEQUENTIAL}
    assert {e for e, _ in reached} == engines, sorted(engines - {e for e, _ in reached})
    # both layouts of the engines that have two, and DistSum rows wider than one pass
    for e, layouts in [("DistF32Generic", {"staged", "direct"}), ("DistI8", {"sub-warp groups", "one row at a time"}),
                       ("DistSum", {"several passes"})]:
        assert {l for x, l in reached if x == e} >= layouts, (e, layouts)


def test_the_builder_parity_list_holds_each_side_of_every_bound():
    engine, _ = engine_choice()
    for kind in ("angular", "angular_int"):
        dims = {dim for k, dim, _, _, _ in SEQUENTIAL if k == kind}
        # the widths where the layout changes: dim - 1 and dim take different layouts of one engine
        edges = [(d - 1, d) for d in range(2, 8192)
                 if engine(kind, d - 1)[0] == engine(kind, d)[0] and engine(kind, d - 1)[1] != engine(kind, d)[1]
                 and engine(kind, d)[1] not in ("tail", "no tail")]
        assert edges, kind
        for lo, hi in edges:
            assert lo in dims and hi in dims, "%s: no builder case at %d and %d (%s / %s)" % (
                kind, lo, hi, engine(kind, lo), engine(kind, hi))
    # i8 rows whose exact r and dx of a saturated row (127 * 127 * dim) no longer fit a float's 24-bit significand
    assert any(127 * 127 * dim > 2 ** 24 for k, dim, _, _, _ in SEQUENTIAL if k == "angular_int")
