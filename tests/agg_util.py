"""Shared inputs of the aggregation tests: toy Groth16 keys with known secrets and proofs made from them, re-randomised
copies of the proof_of_twitter fixture, and the byte layouts zke_prove uses."""
import random

from oracle import bn254 as b
from oracle import aggregate as ag

from test_verifier_fixture import _load

R = b.R
TAU_A, TAU_B = 0x1234567, 0x7654321   # the two secrets of the toy SRS


def toy_key(n_pub: int, seed: int = 1):
    """A Groth16 verification key with known secrets (alpha, beta, gamma, delta, IC scalars)."""
    rnd = random.Random(seed)
    al, be, ga, de = (rnd.randrange(1, R) for _ in range(4))
    ic = [rnd.randrange(1, R) for _ in range(n_pub + 1)]
    vk = {"protocol": "groth16", "curve": "bn128", "nPublic": n_pub,
          "vk_alpha_1": b.g1_to_json(b.g1_mul(b.G1_GEN, al)), "vk_beta_2": b.g2_to_json(b.g2_mul(b.G2_GEN, be)),
          "vk_gamma_2": b.g2_to_json(b.g2_mul(b.G2_GEN, ga)), "vk_delta_2": b.g2_to_json(b.g2_mul(b.G2_GEN, de)),
          "IC": [b.g1_to_json(b.g1_mul(b.G1_GEN, k)) for k in ic]}
    return vk, (al, be, ga, de, ic)


def toy_proof(secrets, pubs, rnd):
    """A valid proof of `pubs` under toy_key's key: A = a g, B = b h, C = (a b - alpha beta - gamma x) / delta g."""
    al, be, ga, de, ic = secrets
    a, bb = rnd.randrange(1, R), rnd.randrange(1, R)
    x = (ic[0] + sum(s * k for s, k in zip(pubs, ic[1:]))) % R
    c = (a * bb - al * be - x * ga) * pow(de, -1, R) % R
    return (b.g1_mul(b.G1_GEN, a), b.g2_mul(b.G2_GEN, bb), b.g1_mul(b.G1_GEN, c))


def toy_batch(n: int, seed: int = 7, n_pub: int = 2):
    vk, sec = toy_key(n_pub)
    rnd = random.Random(seed)
    pubs = [[rnd.randrange(R) for _ in range(n_pub)] for _ in range(n)]
    return vk, sec, pubs, [toy_proof(sec, p, rnd) for p in pubs]


def twitter_batch(n: int, seed: int = 11):
    """n re-randomised copies of the proof_of_twitter fixture: (k A, k^-1 B + s delta, C + s k A)."""
    vkey, public, proof = _load()
    rnd = random.Random(seed)
    a, bb, c = b.g1_from_json(proof["pi_a"]), b.g2_from_json(proof["pi_b"]), b.g1_from_json(proof["pi_c"])
    delta = b.g2_from_json(vkey["vk_delta_2"])
    proofs = []
    for _ in range(n):
        k, s = rnd.randrange(1, R), rnd.randrange(R)
        ka = b.g1_mul(a, k)
        proofs.append((ka, b.g2_add(b.g2_mul(bb, pow(k, -1, R)), b.g2_mul(delta, s)), b.g1_add(c, b.g1_mul(ka, s))))
    return vkey, [[int(x) for x in public]] * n, proofs


def proof_json(p):
    return {"pi_a": b.g1_to_json(p[0]), "pi_b": b.g2_to_json(p[1]), "pi_c": b.g1_to_json(p[2]), "protocol": "groth16"}


def proofs256(proofs) -> bytes:
    return b"".join(ag.g1_b(p[0]) + ag.g2_b(p[1]) + ag.g1_b(p[2]) for p in proofs)


def publics_bytes(pubs) -> bytes:
    return ag.publics_bytes(pubs)
