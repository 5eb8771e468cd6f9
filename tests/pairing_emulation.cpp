// CPU harness for zk-email-verify_b200/csrc/pairing.cuh under ZKE_FF_EMULATE (tests/test_pairing_emulation.py): the
// Fq12 tower operations, the Miller loop (on the fly and replayed from recorded lines), the final exponentiation and
// the G2 subgroup check the batch verifier's kernels run.  All values are Montgomery-form byte images.
#define ZKE_FF_EMULATE
#include "pairing.cuh"
#include <cstring>
#include <vector>
using namespace zke::dev;
extern "C" {
void pe_set_consts(const uint32_t* qmod, const uint32_t* qr, const uint32_t* qr2, uint32_t qinv,
                   const uint32_t* rmod, const uint32_t* rr, const uint32_t* rr2, uint32_t rinv) {
    memcpy(FQ_C.mod, qmod, 32); memcpy(FQ_C.r, qr, 32); memcpy(FQ_C.r2, qr2, 32); FQ_C.inv = qinv;
    memcpy(FR_C.mod, rmod, 32); memcpy(FR_C.r, rr, 32); memcpy(FR_C.r2, rr2, 32); FR_C.inv = rinv;
}
int pe_line_count() { return ATE_LINES; }
// out = op(a[, b]): 0 a*b, 1 a^2, 2 cyclotomic a^2, 3 a^-1, 4/5/6 a^(p^k), 7 a * line(b = l0, l1, l2), 8 final
// exponentiation, 9 conjugate
void pe_f12(int which, const uint8_t* a_bytes, const uint8_t* b_bytes, uint8_t* out) {
    const Fq12 a = Fq12::load(a_bytes);
    Fq12 r;
    switch (which) {
        case 0: r = a * Fq12::load(b_bytes); break;
        case 1: r = a.sqr(); break;
        case 2: r = a.cyclotomic_sqr(); break;
        case 3: r = a.inv(); break;
        case 4: r = a.frobenius<1>(); break;
        case 5: r = a.frobenius<2>(); break;
        case 6: r = a.frobenius<3>(); break;
        case 7: r = a.mul_line(Fq2::load(b_bytes), Fq2::load(b_bytes + 64), Fq2::load(b_bytes + 128)); break;
        case 8: r = final_exponentiation(a); break;
        default: r = a.conj(); break;
    }
    r.store(out);
}
// g1: x, y (64 B); g2: x.c0, x.c1, y.c0, y.c1 (128 B).  out: the Miller loop (final = 0) or the pairing (final = 1)
void pe_pairing(const uint8_t* g1, const uint8_t* g2, int final, uint8_t* out) {
    const G1Affine p = G1Affine::load(g1);
    const G2Affine q = G2Affine::load(g2);
    const Fq12 f = miller_loop<0>(true, q, p, nullptr, nullptr, nullptr);
    (final ? final_exponentiation(f) : f).store(out);
}
// Records the lines of q while computing the Miller loop of (q, p1) on the fly (fly_out), then replays them at p2
// together with the on-the-fly loop of (q2, p3): replay_out = ML(q, p2) ML(q2, p3) computed by the shared-accumulator loop.
void pe_replay(const uint8_t* g1a, const uint8_t* g2a, const uint8_t* g1b, const uint8_t* g2b, const uint8_t* g1c,
               uint8_t* fly_out, uint8_t* replay_out, uint8_t* replay_only_out) {
    std::vector<uint8_t> lines((size_t)LINE_BYTES * ATE_LINES);
    const G1Affine p1 = G1Affine::load(g1a), p2 = G1Affine::load(g1b), p3 = G1Affine::load(g1c);
    const G2Affine q = G2Affine::load(g2a), q2 = G2Affine::load(g2b);
    miller_loop<0>(true, q, p1, nullptr, nullptr, lines.data()).store(fly_out);
    const uint8_t* tab[1] = {lines.data()};
    miller_loop<1>(true, q2, p3, tab, &p2, nullptr).store(replay_out);
    miller_loop<1>(false, q2, p3, tab, &p2, nullptr).store(replay_only_out);
}
int pe_g2_check(const uint8_t* g2) {   // bit 0: on the twist, bit 1: in the order-r subgroup
    const G2Affine q = G2Affine::load(g2);
    const bool on = g2_on_curve(q);
    return (on ? 1 : 0) | (on && g2_in_subgroup(q) ? 2 : 0);
}
}
