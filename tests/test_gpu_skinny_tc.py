"""The batch-sized split-bf16 projections (csrc/skinny_tc.cuh behind mac_linear_tc_small_fwd: projY, the folded write unit
with its y2 / n_split column split, the write gate and ctrlProj) at every form the kernel launches.

Launch rule (skinny_tc_launch, restated in `launch_form`): a CTA owns BN = 64 output columns iff n_out % 64 == 0 and
n_out >= 1024, else 32; at M <= 64 its two warpgroups split the CTA's columns (the column form, m64 n(BN/2)), above that
its rows (the row form); wt_lo == NULL runs the single bf16 pass instead of the three-pass split.  That makes 8 kernel
instances, and FORM_CASES launches each of them (tests/test_skinny_tc_bounds.py asserts so on the CPU).  The fp32
activations arrive by TMA into a ring of 4 stages in the column form and 2 in the row form, beside a weight ring of 6 or 4
stages and the 3-stage bf16 ring: RING_CASES run k-block counts of every remainder mod 12 (which covers all six depths)
and one above 24, with segment boundaries off every ring boundary.

Every call is checked against fp64 of exactly its operands within the bars of tests/test_gpu_wgmma.py, over inputs whose
allocations are NaN below row M and in their ldx padding (the tensor maps must stop at M rows and k columns) and outputs
with NaN guard rows and columns (only rows [0, M) of the owned columns may change); a rerun, and the same call on compact
copies of the inputs, must give the same bits, and inputs and packs must come back bit-unchanged.  Rows are independent
of M bit for bit, across the switch between the two forms too; the column split and the write gate's z equal, bit for
bit, the plain call and the sigmoid call they stand for.  Arguments the kernel cannot serve are refused before any launch
and any write (REFUSALS; their CPU twin is in tests/test_skinny_tc_bounds.py)."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_gpu_wgmma import (ERR_ALIGN, ERR_INVALID, ERR_UNSUPPORTED, TOL_SKINNY_SINGLE, TOL_SKINNY_SPLIT,
                                  TOL_SKINNY_TRUE, act_ref, excess, gen, pack_split, randn, run_skinny, skinny_refs)

pytestmark = pytest.mark.gpu

NAN = float("nan")
GUARD = 2                      # NaN rows above and below every output
BIAS_CONST = {"vec": -0.2, "const": 0.3, "none": 0.0}


def launch_form(M, n_out, split):
    """skinny_tc_launch's choice of kernel instance: (BN, three-pass split, column form)"""
    return (64 if n_out % 64 == 0 and n_out >= 1024 else 32, bool(split), M <= 64)


ALL_FORMS = {(bn, split, cols) for bn in (32, 64) for split in (True, False) for cols in (True, False)}


def case(M, segs, n_out, split=True, bias="vec", act="NON", ldy=None, wide=None, n_split=0, gate=None):
    """One call: segment `wide` is strided (ldx = k + 96), n_split > 0 sends columns >= n_split to y2, gate "z" / "no_z" is
    the write gate with / without gate_z.  ldy defaults to the narrowest the outputs take."""
    if ldy is None:
        ldy = max(n_split, n_out - n_split) if n_split else n_out
    c = dict(M=M, segs=tuple(segs), n_out=n_out, split=split, bias=bias, act=act, ldy=ldy, wide=wide, n_split=n_split,
             gate=gate)
    name = "M%d-k%s-n%d-%s-%s-%s-ldy%d" % (M, "+".join(map(str, segs)), n_out, "split" if split else "single", bias, act,
                                           ldy)
    name += ("-wide%d" % wide if wide is not None else "") + ("-nsplit%d" % n_split if n_split else "")
    name += "-gate_%s" % gate if gate else ""
    return pytest.param(c, id=name)


FORM_CASES = [
    # BN 32, split, column form
    case(37, (64, 64, 128), 96, bias="const", act="TANH", ldy=128, wide=0),
    case(64, (512,), 512, ldy=544, gate="z"),                                  # the write gate at 64 rows
    # BN 32, split, row form
    case(100, (512,), 512, ldy=544, gate="no_z"),                              # the write gate at 100 rows, no gate_z
    case(128, (128, 64, 192, 64), 160, bias="none", act="ELU", n_split=64, ldy=128, wide=2),
    # BN 32, single pass, column form
    case(50, (192, 64), 288, split=False, act="SIGMOID", wide=1),
    # BN 32, single pass, row form
    case(65, (256,), 480, split=False, bias="const", act="RELU_STD", ldy=512),
    # BN 64, split, column form: the headline's folded write unit exactly, then n_split = 17 x 32 between the two
    # warpgroups' column halves of CTA 8
    case(64, (512, 512), 1024, n_split=512, ldy=512),
    case(33, (512, 512), 1024, n_split=544, ldy=576, wide=1),
    # BN 64, split, row form
    case(100, (256, 192, 64), 1024, bias="none", act="RELU_STD", n_split=480, ldy=544, wide=0),
    case(128, (512, 512), 1088, act="TANH"),
    # BN 64, single pass, column form
    case(1, (1024,), 1024, split=False, bias="const", act="ELU"),
    case(64, (64, 448), 1088, split=False, act="TANH", ldy=1152, wide=1),
    # BN 64, single pass, row form
    case(77, (448, 64), 1024, split=False, act="SIGMOID", n_split=352, ldy=672, wide=0),
]

# k-blocks per segment for each k-block count: counts 1..12 take every remainder mod 12 (= lcm of the 4 / 6 / 3 and
# 2 / 4 / 3 ring depths), 29 wraps every ring several times; every boundary sits at a k-block = 1 or 5 (mod 6), on no
# ring's boundary
RING_SEGS = {1: (1,), 2: (1, 1), 3: (1, 2), 4: (1, 3), 5: (1, 4), 6: (1, 4, 1), 7: (1, 4, 2), 8: (1, 4, 2, 1),
             9: (1, 4, 2, 2), 10: (5, 2, 3), 11: (1, 4, 2, 4), 12: (5, 2, 4, 1), 29: (5, 8, 6, 10)}
RING_CASES = [case(M, tuple(64 * b for b in blocks), 1024 if n % 2 else 96, wide=1 if len(blocks) > 1 else None)
              for M in (64, 128) for n, blocks in RING_SEGS.items()]


# ------------------------------------------------------------------------------------------------ operands and checks
def operands(c, seed, device="cuda"):
    """The call's inputs: each segment a [M, k] view of a [128, ldx] allocation that is NaN below row M and in its ldx
    padding; W [K, n_out] with its packs; bias; the write gate's operands [M, ldy]."""
    g = gen(seed) if device == "cuda" else torch.Generator().manual_seed(seed)
    rn = (lambda *s, scale=1.0: randn(g, *s, scale=scale)) if device == "cuda" else \
        (lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale)
    M, n_out, ldy = c["M"], c["n_out"], c["ldy"]
    xs = []
    for i, k in enumerate(c["segs"]):
        ldx, off = (k + 96, 32) if i == c["wide"] else (k, 0)
        buf = torch.full((128, ldx), NAN, device=device)
        buf[:M, off:off + k] = rn(M, k)
        xs.append(buf[:M, off:off + k])
    K = sum(c["segs"])
    W = rn(K, n_out, scale=K ** -0.5)
    hi, lo = pack_split(W) if device == "cuda" else split_pack_cpu(W)
    b = rn(n_out, scale=0.5) if c["bias"] == "vec" else None
    gnew, gold = (rn(M, ldy), rn(M, ldy)) if c["gate"] else (None, None)
    return dict(xs=xs, W=W, hi=hi, lo=lo, b=b, bias_const=BIAS_CONST[c["bias"]], gnew=gnew, gold=gold)


def split_pack_cpu(W):
    """mac_pack_weight_bf16_split's result on the CPU: hi = bf16(W^T), lo = bf16(W^T - hi), both [n_out, K]"""
    hi = W.t().contiguous().to(torch.bfloat16)
    return hi, (W.t().contiguous() - hi.float()).to(torch.bfloat16)


def owned(c):
    """{output: columns the call owns}"""
    n_out, ns = c["n_out"], c["n_split"]
    out = {"y": ns or n_out}
    if ns:
        out["y2"] = n_out - ns
    if c["gate"] == "z":
        out["z"] = n_out
    return out


def launch(c, ops, xs=None):
    """Run call c into fresh NaN buffers [GUARD + M + GUARD, ldy]; returns {output: buffer}."""
    M, ldy = c["M"], c["ldy"]
    bufs = {k: torch.full((M + 2 * GUARD, ldy), NAN, device="cuda") for k in owned(c)}
    view = {k: v[GUARD:GUARD + M] for k, v in bufs.items()}
    gate = (ops["gnew"], ops["gold"], view.get("z")) if c["gate"] else (None, None, None)
    L_.check(run_skinny(ops["xs"] if xs is None else xs, ops["hi"], ops["lo"] if c["split"] else None, ops["b"],
                        ops["bias_const"], c["act"], view["y"], ldy, M, c["n_out"], y2=view.get("y2"),
                        n_split=c["n_split"], gate=gate), "mac_linear_tc_small_fwd")
    return bufs


def check_call(c, ops, y, y2=None, z=None):
    """The outputs of call c (their owned columns, [M, w]) against fp64 of exactly its operands: {check: (excess, bar)}, the
    excess in units of |X| @ |W| + |bias| (tests/test_gpu_wgmma.py `excess`); the split product also against fp64 of the
    fp32 inputs.  The write gate's z = sigmoid(t) moves by at most |dt| / 4, y = new z + old (1 - z) by |new - old| |dz|,
    and their fp32 evaluation adds a few 1e-7."""
    X = torch.cat([x.contiguous() for x in ops["xs"]], 1)
    exact, single, true, absprod = skinny_refs(X, ops["W"], ops["hi"], ops["lo"], ops["b"], ops["bias_const"])
    refs = {"operands": (exact, TOL_SKINNY_SPLIT), "fp32 inputs": (true, TOL_SKINNY_TRUE)} if c["split"] else \
        {"operands": (single, TOL_SKINNY_SINGLE)}
    n_out, res = c["n_out"], {}
    for what, (pre, bar) in refs.items():
        if c["gate"]:
            gn, go = ops["gnew"][:, :n_out].double(), ops["gold"][:, :n_out].double()
            zr = torch.sigmoid(pre)
            dg = (gn - go).abs()
            res["y vs " + what] = (excess(y, gn * zr + go * (1 - zr), 0.25 * absprod * dg,
                                          tiny=3e-7 * dg + 4e-7 * (gn.abs() + go.abs())), bar)
            if z is not None:
                res["z vs " + what] = (excess(z, zr, 0.25 * absprod, tiny=3e-7), bar)
        else:
            r = act_ref(c["act"], pre)
            tiny = 0.0 if c["act"] == "NON" else 1e-6 * r.abs() + 1e-7          # fp32 tanhf / expf / expm1f
            got = torch.cat([y, y2], 1) if c["n_split"] else y
            res["y vs " + what] = (excess(got, r, absprod, tiny=tiny), bar)
    return res


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def run_case(c, seed):
    """Everything this file asks of one call; returns check_call's result."""
    ops = operands(c, seed)
    before = {k: v.clone() for k, v in ops.items() if torch.is_tensor(v)}
    bases = [x._base if x._base is not None else x for x in ops["xs"]]
    bases_before = [t.clone() for t in bases]
    first = launch(c, ops)
    again = launch(c, ops)
    compact = launch(c, ops, xs=[x.contiguous() for x in ops["xs"]])
    torch.cuda.synchronize()
    for k in first:
        assert same_bits(first[k], again[k]), (k, "a rerun differs")
        assert same_bits(first[k], compact[k]), (k, "NaN rows past M or NaN ldx padding changed the result")
    for k, w in owned(c).items():
        keep = torch.ones_like(first[k], dtype=torch.bool)
        keep[GUARD:GUARD + c["M"], :w] = False
        assert bool(torch.isnan(first[k][keep]).all()), (k, "written outside rows [0, M) x its %d columns" % w)
    for k, v in before.items():
        assert same_bits(ops[k], v), (k, "operand changed")
    for t, t0 in zip(bases, bases_before):
        assert same_bits(t, t0), "activation allocation changed"
    out = {k: first[k][GUARD:GUARD + c["M"], :w] for k, w in owned(c).items()}
    return check_call(c, ops, out["y"], out.get("y2"), out.get("z"))


def assert_within(label, res):
    print("skinny %s: %s" % (label, ", ".join("%s %.2e (bar %.0e)" % (k, e, bar) for k, (e, bar) in res.items())))
    for k, (e, bar) in res.items():
        assert e <= bar, (k, e, bar)


# ------------------------------------------------------------------------------------------------ forms and rings
@pytest.mark.parametrize("c", FORM_CASES)
def test_form_matches_fp64(c):
    assert_within((launch_form(c["M"], c["n_out"], c["split"]), c), run_case(c, 7 * c["M"] + c["n_out"] + len(c["segs"])))


@pytest.mark.parametrize("c", RING_CASES)
def test_ring_remainders_match_fp64(c):
    assert_within((launch_form(c["M"], c["n_out"], c["split"]), c), run_case(c, 13 * c["M"] + sum(c["segs"])))


# ------------------------------------------------------------------------------------------------ bit-for-bit identities
@pytest.mark.parametrize("n_out,split", [(512, True), (1024, True), (512, False), (1024, False)])
def test_rows_are_independent_of_m(n_out, split):
    """X[128, K] and W fixed, every M from 1 to 128: rows [0, M) are the bits of M = 64 in the column form and of M = 128
    in the row form, and the two forms agree on rows [0, 64)."""
    g = gen(n_out + split)
    segs = (256, 192)                     # 7 k-blocks, the boundary inside a ring
    X = [randn(g, 128, k) for k in segs]
    W = randn(g, sum(segs), n_out, scale=sum(segs) ** -0.5)
    hi, lo = pack_split(W)
    b = randn(g, n_out, scale=0.5)
    ys = {}
    for M in range(1, 129):
        ys[M] = torch.full((128, n_out), NAN, device="cuda")
        L_.check(run_skinny([x[:M] for x in X], hi, lo if split else None, b, 0.1, "ELU", ys[M], n_out, M, n_out))
    torch.cuda.synchronize()
    for M, y in ys.items():
        top = 64 if M <= 64 else 128
        assert same_bits(y[:M], ys[top][:M]), (M, top)
        assert bool(torch.isnan(y[M:]).all()), M
    assert same_bits(ys[64][:64], ys[128][:64]), "the column form (M <= 64) and the row form differ on rows [0, 64)"
    c = dict(segs=segs, n_out=n_out, split=split, act="ELU", gate=None, n_split=0)
    ops = dict(xs=X, W=W, hi=hi, lo=lo, b=b, bias_const=0.1)
    assert_within(("rows", n_out, split), check_call(c, ops, ys[128]))


@pytest.mark.parametrize("M,n_out,n_split,ldy", [(64, 1024, 512, 512), (33, 1024, 544, 544), (100, 1024, 544, 576),
                                                  (128, 512, 224, 320), (7, 512, 96, 416)])
def test_column_split_equals_the_unsplit_call(M, n_out, n_split, ldy):
    """y[:, :n_split] and y2[:, :n_out - n_split] are, bit for bit, the columns of the same call without y2."""
    c = dict(M=M, segs=(512, 512), n_out=n_out, split=True, bias="vec", act="TANH", ldy=n_out, wide=None, n_split=0,
             gate=None)
    ops = operands(c, M + n_split)
    full = launch(c, ops)["y"][GUARD:GUARD + M]
    c.update(ldy=ldy, n_split=n_split)
    parts = launch(c, ops)
    torch.cuda.synchronize()
    assert same_bits(parts["y"][GUARD:GUARD + M, :n_split], full[:, :n_split])
    assert same_bits(parts["y2"][GUARD:GUARD + M, :n_out - n_split], full[:, n_split:])


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("M", [1, 64, 100, 128])
def test_gate_z_equals_the_sigmoid_call(M, split):
    """The write gate's z is, bit for bit, the SIGMOID call with the same bias (both sigmoid_f), and its y does not depend
    on whether z is stored."""
    c = dict(M=M, segs=(512,), n_out=512, split=split, bias="vec", act="NON", ldy=544, wide=None, n_split=0, gate="z")
    ops = operands(c, 3 * M + split)
    with_z = launch(c, ops)
    without_z = launch(dict(c, gate="no_z"), ops)
    sig = launch(dict(c, gate=None, act="SIGMOID"), ops)
    torch.cuda.synchronize()
    assert same_bits(with_z["z"], sig["y"])
    assert same_bits(with_z["y"], without_z["y"])


# ------------------------------------------------------------------------------------------------ refusals
def refusal(expect, M=8, segs=((64, 64),), n_out=64, ldy=64, n_split=None, gate=None, odd=(), why=""):
    """A call the library must refuse: segs (k, ldx) per segment; n_split not None passes y2; gate "new_only", "z_only"
    (gate_z without the gate) or "z" (the whole gate); `odd` names the pointers placed 8 bytes off 16-byte alignment."""
    return pytest.param(dict(M=M, segs=segs, n_out=n_out, ldy=ldy, n_split=n_split, gate=gate, odd=odd), expect, id=why)


REFUSALS = [
    refusal(ERR_INVALID, M=129, why="M>128"),
    refusal(ERR_INVALID, M=0, why="M=0"),
    refusal(ERR_UNSUPPORTED, n_out=48, ldy=48, why="n_out%32"),
    refusal(ERR_UNSUPPORTED, segs=((96, 96),), why="k%64"),
    refusal(ERR_INVALID, ldy=32, why="ldy<n_out"),
    refusal(ERR_INVALID, ldy=0, why="ldy=0"),
    refusal(ERR_INVALID, n_split=0, ldy=64, why="y2-n_split=0"),
    refusal(ERR_INVALID, n_split=-32, ldy=64, why="y2-n_split<0"),
    refusal(ERR_INVALID, n_split=64, ldy=64, why="y2-n_split=n_out"),
    refusal(ERR_INVALID, n_split=96, ldy=96, why="y2-n_split>n_out"),
    refusal(ERR_INVALID, n_out=128, n_split=96, ldy=64, why="y2-ldy<n_split"),
    refusal(ERR_INVALID, n_out=128, n_split=32, ldy=64, why="y2-ldy<n_out-n_split"),
    refusal(ERR_UNSUPPORTED, n_split=16, ldy=64, why="y2-n_split%32"),
    refusal(ERR_INVALID, segs=((64, 32),), why="ldx<k"),
    refusal(ERR_INVALID, segs=((64, -64),), why="ldx<0"),
    refusal(ERR_INVALID, segs=((64, 64), (128, 64)), why="second-segment-ldx<k"),
    refusal(ERR_UNSUPPORTED, n_split=32, gate="z", why="gate-with-y2"),
    refusal(ERR_INVALID, gate="z_only", why="gate_z-without-gate"),
    refusal(ERR_INVALID, gate="new_only", why="gate_new-without-gate_old"),
    refusal(ERR_ALIGN, odd=("x",), why="odd-x"),
    refusal(ERR_ALIGN, odd=("lo",), why="odd-wt_lo"),
    refusal(ERR_ALIGN, n_split=32, ldy=32, odd=("y2",), why="odd-y2"),
    refusal(ERR_ALIGN, gate="z", odd=("z",), why="odd-gate_z"),
    refusal(ERR_ALIGN, gate="z", odd=("old",), why="odd-gate_old"),
]


def call_refused(lib, r, ops, out, stream=None):
    """r with every operand at address `ops` and every output at address `out` (each + 8 where r misaligns it)."""
    at = lambda name, base: base + (8 if name in r["odd"] else 0)
    n = len(r["segs"])
    arr_p = (ctypes.c_void_p * n)(*[at("x", ops)] * n)
    arr_k = (ctypes.c_int * n)(*[k for k, _ in r["segs"]])
    arr_ld = (ctypes.c_int * n)(*[ld for _, ld in r["segs"]])
    gate = r["gate"]
    gn = at("new", ops) if gate in ("z", "new_only") else None
    go = at("old", ops) if gate == "z" else None
    gz = at("z", out) if gate in ("z", "z_only") else None
    y2 = at("y2", out) if r["n_split"] is not None else None
    return lib.mac_linear_tc_small_fwd(arr_p, arr_k, arr_ld, n, at("hi", ops), at("lo", ops), None, 0.0, 0, at("y", out),
                                       r["ldy"], y2, r["n_split"] or 0, gn, go, gz, r["M"], r["n_out"], stream)


@pytest.mark.parametrize("r,expect", REFUSALS)
def test_refused_before_any_launch_or_write(r, expect):
    """device buffers: the status, no launch, every operand still zero and every output still NaN"""
    lib = L_.load()
    ops = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.full((1 << 18,), NAN, device="cuda")
    torch.cuda.synchronize()
    before = lib.mac_b200_launch_count()
    st = call_refused(lib, r, ops.data_ptr(), out.data_ptr(), L_.stream_ptr())
    torch.cuda.synchronize()
    assert st == expect, st
    assert lib.mac_b200_launch_count() == before
    assert not bool(ops.any()) and bool(out.isnan().all())
