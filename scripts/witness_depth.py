"""CPU-side analysis of the witness program the engine builds at open time (csrc/witness_program.cpp, reported by
zke_circuit_program_stats): the number of levels and of 512-op iterations left after the native SHA-256 and regex-seeding
substitutions - what the level-synchronous witness kernel (witness.cu) walks, here for one CTA per email.
    python scripts/witness_depth.py [Template p1,p2,...]"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "zk-email-verify_b200", "host"))
import zkemail_b200 as z

T = 512


def analyse(c, native_sha=True, native_rx=True):
    """(levels, iterations, ops that are not cooperative ops, {level: such ops})"""
    st = c.program_stats(native_sha=native_sha, native_regex=native_rx, cluster=1)
    counts = {l + 1: n for l, n in enumerate(st["level_ops"])}
    return st["n_levels"], st["n_iters"], st["n_ops_kept"], counts


if __name__ == "__main__":
    name, params = "EmailVerifier", [1024, 1536, 121, 17]
    if len(sys.argv) > 1:
        name = sys.argv[1]; params = [int(x) for x in sys.argv[2].split(",")] if len(sys.argv) > 2 else []
    c = z.Circuit(name, params)
    for sha_on, rx_on in ((False, False), (True, False), (True, True)):
        depth, iters, kept, counts = analyse(c, sha_on, rx_on)
        thin = sum(1 for l, n in counts.items() if n < T // 4)
        print("native sha %d, regex seeding %d: %7d ops kept, %6d levels, %6d iterations of %d ops (floor %d), %d levels with < %d ops"
              % (sha_on, rx_on, kept, depth, iters, T, -(-kept // T), thin, T // 4))
