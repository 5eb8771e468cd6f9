"""Circom-shaped `.r1cs` images of a chosen domain size, with satisfying witnesses whose values and points are laid out to
reach the prover's edge cases.  The bulk is written with numpy, so a 2^20-row instance takes seconds.

Row kinds:
  free rows       w_f * 1 = w_f            hold for any w_f, so the bulk's values are chosen freely
  quadratic rows  x * y = z                genuine products: the quotient polynomial is not trivial
  shared rows     (sum u_i) * 1 = sum u_i  and  1 * (sum u_i) = sum u_i: every u_i gets the same A, B1, B2 and C points
  opposite rows   the same with p - q:     q's points are the negatives of p's
  A-only rows     x * () = ()              empty B and C: x has points in A only (infinity in B1, B2, C)
  unused wires    in no row                points at infinity everywhere

Wires: [1, output, public input, private input, shared-row wires, opposite pairs, A-only, unused, single-term rows]."""
import numpy as np

from test_r1cs_reader import R, body, container, header

N_OUT, N_PUB, N_PRV = 1, 1, 1
N_PUBLIC = N_OUT + N_PUB

# The witness MSMs (msm.cu: msm_config_witness) sort entries in chunks of 32 and reduce a heavy bucket in up to two extra
# passes of fan-in 32: a window-0 bucket needs both passes above 32 * 32 * 32 = 32 768 entries.
HEAVY_BUCKET = 32 * 32 * 32
SMALL = 7                                 # the repeated small scalar of the shared rows (one window-0 bucket at c = 8)
F_SHARED = 0x0123456789ABCDEF_FEDCBA9876543210_0F1E2D3C4B5A6978_8796A5B4C3D2E1F0 % R
F_OPPOSITE = 0x1BADC0DE_DEADBEEF_CAFEF00D_0BADF00D_12345678_9ABCDEF0_0FEDCBA9_87654321 % R


def window_ones(c):
    """The largest value below r whose c-bit windows are all ones: its signed digits carry through every window."""
    return (1 << (c * (253 // c))) - 1


# values placed on single free rows
SPECIAL = ([0, 1, 2, R - 1, R - 2, (R - 1) // 2, (R + 1) // 2, (R - 3) // 2, (R + 3) // 2]
           + [(1 << k) - 1 for k in (8, 12, 16, 17, 20, 32, 64, 128, 200, 252, 253)]
           + [1 << k for k in (8, 17, 20, 128, 252, 253)]
           + [window_ones(c) for c in (8, 12, 17, 20)])
OPPOSITE_SCALARS = [1, SMALL, F_OPPOSITE, R - 1, (R - 1) // 2, (R + 1) // 2]
A_ONLY = [0, 1, SMALL, R - 1, F_SHARED, 1 << 200]
UNUSED = [1, SMALL, R - 1, F_SHARED, (R + 1) // 2, 3]

_ROW = np.dtype([("na", "<u4"), ("wa", "<u4"), ("ca", "u1", 32), ("nb", "<u4"), ("wb", "<u4"), ("cb", "u1", 32),
                 ("nc", "<u4"), ("wc", "<u4"), ("cc", "u1", 32)])


def _limbs(v):
    return [(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]


def rows_for(domain_log2):
    """A row count that lands in 2^domain_log2 (Circuit.domain_log2: smallest k with 2^k >= rows + public + 1), three
    quarters full."""
    n = 1 << domain_log2
    return n - n // 4 - N_PUBLIC - 1


def generate(domain_log2, seed=1, heavy=True):
    """{"blob": .r1cs image, "witness": bytes, "values": (n_wires, 4) uint64 limbs, "n_wires", "n_rows", "classes":
    name -> wire indices, "quad_rows": the quadratic rows, in the order of classes["quadratic"]}.  heavy: the shared rows carry more than HEAVY_BUCKET wires of one small scalar."""
    rng = np.random.default_rng(seed)
    n_rows = rows_for(domain_log2)
    nxt = 1 + N_OUT + N_PUB + N_PRV
    classes = {}

    def fresh(k):
        nonlocal nxt
        nxt += k
        return np.arange(nxt - k, nxt, dtype=np.int64)

    explicit = {}                      # wire -> value, for everything outside the numpy-drawn bulk
    rows = []                          # multi-term rows, written with test_r1cs_reader.body

    # shared rows: identical points; scalars 1 (the ones list), one full-width value, and the small value (one bucket)
    n_small = HEAVY_BUCKET + 200 if heavy else 32
    ident = fresh(16 + 16 + n_small)
    classes["identical_one"], classes["identical_full"], classes["identical_small"] = ident[:16], ident[16:32], ident[32:]
    for w in ident:
        explicit[int(w)] = 1 if w < ident[16] else (F_SHARED if w < ident[32] else SMALL)
    lc = [(int(w), 1) for w in ident]
    rows += [(lc, [(0, 1)], lc), ([(0, 1)], lc, lc)]

    # opposite rows: one pair per row pair for each scalar, then eight pairs sharing one row pair
    pairs = []
    for v in OPPOSITE_SCALARS + [5] * 8:
        p, q = (int(w) for w in fresh(2))
        explicit[p] = explicit[q] = v
        pairs.append((p, q))
    for p, q in pairs[:len(OPPOSITE_SCALARS)]:
        lc = [(p, 1), (q, R - 1)]
        rows += [(lc, [(0, 1)], lc), ([(0, 1)], lc, lc)]
    lc = [t for p, q in pairs[len(OPPOSITE_SCALARS):] for t in ((p, 1), (q, R - 1))]
    rows += [(lc, [(0, 1)], lc), ([(0, 1)], lc, lc)]
    classes["opposite_p"] = np.array([p for p, _ in pairs])
    classes["opposite_q"] = np.array([q for _, q in pairs])

    a_only = fresh(len(A_ONLY))
    for w, v in zip(a_only, A_ONLY):
        explicit[int(w)] = v
        rows.append(([(int(w), 1)], [], []))
    classes["a_only"] = a_only
    unused = fresh(len(UNUSED))
    for w, v in zip(unused, UNUSED):
        explicit[int(w)] = v
    classes["unused"] = unused

    # single-term rows: the signals, the special values, quadratic rows spread evenly, free rows
    n_single = n_rows - len(rows)
    n_quad = max(8, n_single // 64)
    n_free = n_single - n_quad
    assert n_free >= 3 + len(SPECIAL), "domain too small for the fixed rows"
    special = fresh(len(SPECIAL))
    for w, v in zip(special, SPECIAL):
        explicit[int(w)] = v
    classes["special"] = special
    quad = fresh(3 * n_quad).reshape(n_quad, 3)
    for x, y, zz in quad:
        a, b = (int.from_bytes(rng.bytes(32), "little") % R for _ in range(2))
        explicit[int(x)], explicit[int(y)], explicit[int(zz)] = a, b, a * b % R
    classes["quadratic"] = quad
    bulk = fresh(n_free - 3 - len(SPECIAL))
    free = np.concatenate([np.arange(1, 1 + N_OUT + N_PUB + N_PRV), special, bulk])
    n_wires = nxt

    vals = np.zeros((n_wires, 4), dtype=np.uint64)
    vals[0, 0] = 1
    # the bulk: mostly bits (as in EmailVerifier), then small values, then full-width values below 2^253
    u = rng.random(len(bulk))
    bit, small = u < 0.7, (u >= 0.7) & (u < 0.85)
    full = ~(bit | small)
    vals[bulk[bit], 0] = rng.integers(0, 2, int(bit.sum()), dtype=np.uint64)
    vals[bulk[small], 0] = rng.integers(2, 256, int(small.sum()), dtype=np.uint64)
    vals[bulk[full]] = rng.integers(0, 1 << 64, (int(full.sum()), 4), dtype=np.uint64, endpoint=False)
    vals[bulk[full], 3] &= np.uint64((1 << 61) - 1)
    for w in range(1, 1 + N_OUT + N_PUB + N_PRV):
        explicit[w] = (F_SHARED * w) % R
    for w, v in explicit.items():
        vals[w] = _limbs(v)
    classes["bit"], classes["small"], classes["full_width"] = bulk[bit], bulk[small], bulk[full]

    single = np.zeros(n_single, dtype=_ROW)
    single["na"] = single["nb"] = single["nc"] = 1
    single["ca"][:, 0] = single["cb"][:, 0] = single["cc"][:, 0] = 1
    at_quad = np.zeros(n_single, dtype=bool)
    at_quad[np.linspace(0, n_single - 1, n_quad).astype(np.int64)] = True
    single["wa"][at_quad], single["wb"][at_quad], single["wc"][at_quad] = quad[:, 0], quad[:, 1], quad[:, 2]
    single["wa"][~at_quad], single["wb"][~at_quad], single["wc"][~at_quad] = free, 0, free

    hdr = header(n_wires, n_rows, n_wires, n_out=N_OUT, n_pub=N_PUB, n_prv=N_PRV)
    blob = container([(1, hdr), (2, body(rows) + single.tobytes())])
    return {"blob": blob, "witness": vals.tobytes(), "values": vals, "n_wires": n_wires, "n_rows": n_rows,
            "classes": classes, "quad_rows": len(rows) + np.flatnonzero(at_quad)}


def value(g, wire):
    return sum(int(x) << (64 * i) for i, x in enumerate(g["values"][wire]))
