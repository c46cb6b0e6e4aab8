"""TEST INFRASTRUCTURE - the reference's PlonkVersion matrix restated on top of oracle/pyref.py and oracle/verify.py.

- The legacy transcript seed (Transcript::base + VerifierKey::seed_transcript_legacy, transcript.rs:110-129,
  widget.rs:218-265) is the V3 seed with the commitment of s_sigma_1 appended under the "s_sigma_4" label.
- `prove(..., version)`: V3 is pyref.prove.  V2 is pyref.prove under the legacy seed (Prover::prove_inner reads the
  version only in transcript_for_version, prover.rs:404-430).  V1 also uses the pre-fix opening at z: W_z aggregates
  [r, a, b, c, d, s_sigma_1, s_sigma_2, s_sigma_3], the list forge_proof uses (proof.rs:1637-1650).  The reference
  refuses to make V1 proofs; this one exists only to make V1-valid test proofs.
- `right_and_left` / `verify_with_secret(..., version)`: Proof::verify (V2, V3) and Proof::verify_legacy (V1,
  proof.rs:518-790) with the final pairing replaced by the G1 identity under the known SRS secret, as
  oracle/verify.py does for V3.
- `forge_proof`: the reference's soundness test (proof.rs:1332-1682): honest wires, a random permutation polynomial,
  random quotient chunks, a q_arith evaluation solved after z is known, the legacy seed and the legacy opening.  V1
  accepts it because V1 does not bind the selector evaluations; V2 and V3 reject it.

Only tests/ may import this file."""
from __future__ import annotations

import dataclasses
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

from oracle import pyref as P
from oracle import verify as OV

R_MOD = P.R_MOD
VERSIONS = (1, 2, 3)


def _legacy_comms(comms: Dict[str, object]) -> Dict[str, object]:
    return {**comms, "s_sigma_4": comms["s_sigma_1"]}


def base_transcript(label: bytes, constraints: int, key_comms: Dict[str, object], version: int) -> P.Transcript:
    """Transcript::base_v3 (V3) or Transcript::base (V1, V2), seeded; key_comms by pyref.POLY_NAMES name."""
    assert version in VERSIONS
    comms = key_comms if version == 3 else _legacy_comms(key_comms)
    return P.base_transcript_v3(SimpleNamespace(label=label, constraints=constraints, comms=comms))


def aggregate_witness(polys: Sequence[Sequence[int]], point: int, v: int) -> List[int]:
    """CommitKey::compute_aggregate_witness (key.rs:394-417)."""
    coeffs = [0] * max(len(p) for p in polys)
    power = 1
    for p in polys:
        for i, t in enumerate(p):
            coeffs[i] = (coeffs[i] + t * power) % R_MOD
        power = power * v % R_MOD
    return P.ruffini(P.poly_trim(coeffs), point)


def prove(pd: P.ProverData, rng: P.StdRng, comp: P.Composer, version: int = 3, trace: Optional[P.ProofTrace] = None) -> bytes:
    """A proof under `version`; the same RNG draws as pyref.prove for every version."""
    assert version in VERSIONS
    if version == 3:
        return P.prove(pd, rng, comp, trace)
    trace = trace if trace is not None else P.ProofTrace()
    proof = P.prove(dataclasses.replace(pd, comms=_legacy_comms(pd.comms)), rng, comp, trace)
    if version == 2:
        return proof
    t = trace.values
    w_z = aggregate_witness([t["r_poly"], *t["wire_polys"], *(pd.polys[f"s_sigma_{j}"] for j in (1, 2, 3))], t["z_challenge"], t["v_challenge"])
    w_z_comm = P.commit(pd.commit_key, w_z)
    t.update(w_z=w_z, w_z_comm=w_z_comm)
    out = proof[: 48 * 9] + P.g1_compress(w_z_comm) + proof[48 * 10 :]
    trace.proof_bytes = out
    return out


def challenges(proof: bytes, label: bytes, constraints: int, key_comms, pi_vals: Sequence[int], version: int) -> Dict[str, int]:
    """The transcript replay of Proof::verify / verify_legacy (identical after the seed, proof.rs:237-311, 540-614)."""
    comm, e = OV.parse_proof(proof)
    t = base_transcript(label, constraints, key_comms, version)
    for pi in pi_vals:
        t.append_scalar(b"pi", pi % R_MOD)
    for k in ("a", "b", "c", "d"):
        t.append_commitment(k.encode() + b"_comm", comm[k])
    c = {}
    c["beta"] = t.challenge_scalar(b"beta")
    t.append_scalar(b"beta", c["beta"])
    c["gamma"] = t.challenge_scalar(b"gamma")
    t.append_commitment(b"z_comm", comm["z"])
    c["alpha"] = t.challenge_scalar(b"alpha")
    c["range"] = t.challenge_scalar(b"range separation challenge")
    c["logic"] = t.challenge_scalar(b"logic separation challenge")
    c["fixed"] = t.challenge_scalar(b"fixed base separation challenge")
    c["var"] = t.challenge_scalar(b"variable base separation challenge")
    for k in ("t_low", "t_mid", "t_high", "t_fourth"):
        t.append_commitment(k.encode() + b"_comm", comm[k])
    c["z"] = t.challenge_scalar(b"z_challenge")
    for lab, k in ((b"a_eval", "a"), (b"b_eval", "b"), (b"c_eval", "c"), (b"d_eval", "d"), (b"s_sigma_1_eval", "s1"),
                   (b"s_sigma_2_eval", "s2"), (b"s_sigma_3_eval", "s3"), (b"z_eval", "z"), (b"a_w_eval", "a_w"),
                   (b"b_w_eval", "b_w"), (b"d_w_eval", "d_w"), (b"q_arith_eval", "q_arith"), (b"q_c_eval", "q_c"),
                   (b"q_l_eval", "q_l"), (b"q_r_eval", "q_r")):
        t.append_scalar(lab, e[k])
    c["v"] = t.challenge_scalar(b"v_challenge")
    c["v_w"] = t.challenge_scalar(b"v_w_challenge")
    t.append_commitment(b"w_z_chall_comm", comm["w_z"])
    t.append_commitment(b"w_z_chall_w_comm", comm["w_zw"])
    c["u"] = t.challenge_scalar(b"u_challenge")
    return c


def right_and_left(proof: bytes, label: bytes, constraints: int, key_comms, pi_idx: Sequence[int], pi_vals: Sequence[int],
                   g, version: int):
    """The two G1 points of the final pairing check: right_projective = z W_z + u z w W_zw + [F] - [E] and
    W_z + u W_zw (proof.rs:452-512 for V2 and V3, 742-760 for V1).  None when z lies in the domain."""
    comm, e = OV.parse_proof(proof)
    c = challenges(proof, label, constraints, key_comms, pi_vals, version)
    alpha, beta, gamma, z_ch, v, v_w, u = c["alpha"], c["beta"], c["gamma"], c["z"], c["v"], c["v_w"], c["u"]
    n = 1 << (constraints - 1).bit_length() if constraints > 1 else 1
    domain = P.EvaluationDomain(n)
    z_h = domain.evaluate_vanishing_polynomial(z_ch)
    if (z_ch - 1) % R_MOD == 0:
        return None
    l1 = z_h * P.fr_inv(n * (z_ch - 1) % R_MOD) % R_MOD
    w_inv = P.fr_inv(domain.group_gen)
    pi_eval = 0
    for idx, val in zip(pi_idx, pi_vals):
        if val % R_MOD == 0:
            continue
        den = (pow(w_inv, idx, R_MOD) * z_ch - 1) % R_MOD
        if den == 0:
            return None
        pi_eval = (pi_eval + val * P.fr_inv(den)) % R_MOD
    pi_eval = pi_eval * z_h % R_MOD * P.fr_inv(n) % R_MOD
    r0 = (pi_eval - l1 * alpha * alpha
          - alpha * (e["a"] + beta * e["s1"] + gamma) * (e["b"] + beta * e["s2"] + gamma) % R_MOD
          * (e["c"] + beta * e["s3"] + gamma) % R_MOD * (e["d"] + gamma) % R_MOD * e["z"]) % R_MOD

    K = key_comms
    # the evaluations opened at z: V_MAX_DEGREE = 11 (V2, V3) or V_MAX_DEGREE_LEGACY = 7 (V1), then a_w, b_w, d_w
    at_z = ["a", "b", "c", "d", "s1", "s2", "s3"] + ([] if version == 1 else ["q_arith", "q_c", "q_l", "q_r"])
    at_z_points = [comm["a"], comm["b"], comm["c"], comm["d"], K["s_sigma_1"], K["s_sigma_2"], K["s_sigma_3"]]
    if version != 1:
        at_z_points += [K["q_arith"], K["q_c"], K["q_l"], K["q_r"]]
    V = len(at_z)
    vc = [v]
    for _ in range(1, V):
        vc.append(vc[-1] * v % R_MOD)
    vc.append(v_w * u % R_MOD)
    vc.append(vc[V] * v_w % R_MOD)
    vc.append(vc[V + 1] * v_w % R_MOD)
    E = (sum(e[k] * s for k, s in zip(at_z + ["a_w", "b_w", "d_w"], vc)) - r0 + u * e["z"]) % R_MOD

    scalars: List[int] = []
    points: List[object] = []

    def term(s, p):
        scalars.append(s % R_MOD)
        points.append(p)

    # append_linearization_commitment_terms: shared by every version
    term(e["a"] * e["b"] * e["q_arith"], K["q_m"])
    term(e["a"] * e["q_arith"], K["q_l"])
    term(e["b"] * e["q_arith"], K["q_r"])
    term(e["c"] * e["q_arith"], K["q_o"])
    term(e["d"] * e["q_arith"], K["q_f"])
    term(e["q_arith"], K["q_c"])
    term(P.widget_range_scalar(c["range"], e["a"], e["b"], e["c"], e["d"], e["d_w"]), K["q_range"])
    term(P.widget_logic_scalar(c["logic"], e["q_c"], e["a"], e["a_w"], e["b"], e["b_w"], e["c"], e["d"], e["d_w"]), K["q_logic"])
    term(P.widget_fixed_base_scalar(c["fixed"], e["q_l"], e["q_r"], e["q_c"], e["a"], e["a_w"], e["b"], e["b_w"], e["c"], e["d"], e["d_w"]),
         K["q_fixed_group_add"])
    term(P.widget_curve_add_scalar(c["var"], e["a"], e["a_w"], e["b"], e["b_w"], e["c"], e["d"], e["d_w"]), K["q_variable_group_add"])
    bz = beta * z_ch % R_MOD
    xs = (e["a"] + bz + gamma) * (e["b"] + P.K1 * bz + gamma) % R_MOD * (e["c"] + P.K2 * bz + gamma) % R_MOD \
        * ((e["d"] + P.K3 * bz + gamma) * alpha % R_MOD) % R_MOD
    term(xs + l1 * alpha * alpha + u, comm["z"])
    ys = (e["a"] + beta * e["s1"] + gamma) * (e["b"] + beta * e["s2"] + gamma) % R_MOD * (e["c"] + beta * e["s3"] + gamma) % R_MOD \
        * (beta * e["z"] % R_MOD * alpha % R_MOD) % R_MOD
    term(-ys, K["s_sigma_4"])
    z_pow_n = (z_h + 1) % R_MOD
    for j, k in enumerate(("t_low", "t_mid", "t_high", "t_fourth")):
        term(pow(z_pow_n, j, R_MOD) * -z_h, comm[k])
    # [F], with the shifted openings grouped into a, b and d
    f = vc[:V]
    f[0] = (f[0] + vc[V]) % R_MOD
    f[1] = (f[1] + vc[V + 1]) % R_MOD
    f[3] = (f[3] + vc[V + 2]) % R_MOD
    for s, p in zip(f, at_z_points):
        term(s, p)
    term(-E, g)
    term(z_ch, comm["w_z"])
    term(u * z_ch % R_MOD * domain.group_gen, comm["w_zw"])
    return OV._msm(points, scalars), OV._msm([comm["w_z"], comm["w_zw"]], [1, u])


def verify_with_secret(proof: bytes, label: bytes, constraints: int, key_comms, pi_idx, pi_vals, g, x: int, version: int = 3) -> bool:
    """Verifier::verify_with_version with the pairing replaced by right == [x] left (see oracle/verify.py)."""
    pts = right_and_left(proof, label, constraints, key_comms, pi_idx, pi_vals, g, version)
    if pts is None:
        return False
    right, left = pts
    want = None if left is None else P.jac_to_affine(P.jac_mul(P.jac_from_affine(left), x % R_MOD))
    return right == want


def v1_from_v2_with_secret(proof: bytes, label: bytes, constraints: int, key_comms, pi_vals, g, x: int) -> bytes:
    """The V1 proof of a V2 proof's witness, from the V2 proof's bytes and the SRS secret.  V1 and V2 share the
    seed and every challenge the prover draws; only W_z differs: V2's aggregates q_arith, q_c, q_l and q_r with
    v^8 .. v^11 besides V1's eight polynomials.  Each such term is [(q(X) - q(z)) / (X - z)] =
    (x - z)^-1 ([q] - q(z) g), so V1's W_z needs no polynomial.  Equals prove(..., version=1) for the same RNG."""
    comm, e = OV.parse_proof(proof)
    c = challenges(proof, label, constraints, key_comms, pi_vals, 2)
    inv = P.fr_inv((x - c["z"]) % R_MOD)
    w_z = P.jac_from_affine(comm["w_z"])
    for k, name in enumerate(("q_arith", "q_c", "q_l", "q_r")):
        q = OV._msm([key_comms[name], g], [1, -e[name]])
        if q is not None:
            w_z = P.jac_add(w_z, P.jac_mul(P.jac_from_affine(q), (-pow(c["v"], 8 + k, R_MOD) * inv) % R_MOD))
    return proof[: 48 * 9] + P.g1_compress(P.jac_to_affine(w_z)) + proof[48 * 10 :]


# ---- the reference's soundness test (proof.rs:1298-1743) --------------------------------------------------------
def arith_circuit(comp: P.Composer, a: int, b: int, d: int, public: int) -> None:
    """ArithCircuit (proof.rs:1298-1330): a + b + a b + d + public + 1 = result, then result asserted equal to the
    gate's output."""
    w_a, w_b, w_d = comp.append_witness(a), comp.append_witness(b), comp.append_witness(d)
    w_result = comp.append_witness((a + b + a * b + d + public + 1) % R_MOD)
    out = comp.gate_evaluated(dict(q_l=1, q_r=1, q_m=1, q_f=1, q_c=1), a=w_a, b=w_b, d=w_d, public=public)
    comp.assert_equal(w_result, out)


def linearisation_poly(pd: P.ProverData, ch: Dict[str, int], e: Dict[str, int], z_ch: int, z_poly, t_polys, public_inputs) -> List[int]:
    """linearization_poly::compute (linearization_poly.rs:168-231), as pyref.prove's round 5 forms it."""
    Pp, size = pd.polys, pd.size
    domain = P.EvaluationDomain(size)
    alpha, beta, gamma = ch["alpha"], ch["beta"], ch["gamma"]
    r = P.poly_scale(Pp["q_m"], e["a"] * e["b"] % R_MOD)
    for k, w in (("q_l", "a"), ("q_r", "b"), ("q_o", "c"), ("q_f", "d")):
        r = P.poly_add(r, P.poly_scale(Pp[k], e[w]))
    r = P.poly_scale(P.poly_add(r, Pp["q_c"]), e["q_arith"])
    r = P.poly_add(r, P.poly_scale(Pp["q_range"], P.widget_range_scalar(ch["range"], e["a"], e["b"], e["c"], e["d"], e["d_w"])))
    r = P.poly_add(r, P.poly_scale(Pp["q_logic"], P.widget_logic_scalar(ch["logic"], e["q_c"], e["a"], e["a_w"], e["b"], e["b_w"], e["c"], e["d"], e["d_w"])))
    r = P.poly_add(r, P.poly_scale(Pp["q_fixed_group_add"], P.widget_fixed_base_scalar(ch["fixed"], e["q_l"], e["q_r"], e["q_c"], e["a"], e["a_w"], e["b"],
                                                                                       e["b_w"], e["c"], e["d"], e["d_w"])))
    r = P.poly_add(r, P.poly_scale(Pp["q_variable_group_add"], P.widget_curve_add_scalar(ch["var"], e["a"], e["a_w"], e["b"], e["b_w"], e["c"], e["d"], e["d_w"])))
    r = P.poly_add(r, [P.compute_barycentric_eval(public_inputs, z_ch, domain)])
    bz = beta * z_ch % R_MOD
    s_ident = (e["a"] + bz + gamma) * (e["b"] + P.K1 * bz + gamma) % R_MOD * (e["c"] + P.K2 * bz + gamma) % R_MOD \
        * (e["d"] + P.K3 * bz + gamma) % R_MOD * alpha % R_MOD
    s_copy = (e["a"] + beta * e["s1"] + gamma) * (e["b"] + beta * e["s2"] + gamma) % R_MOD * (e["c"] + beta * e["s3"] + gamma) % R_MOD \
        * (beta * e["z"] % R_MOD) % R_MOD * alpha % R_MOD
    l1_z = P.EvaluationDomain(len(z_poly) - 1 - 2).first_lagrange_coefficient(z_ch)
    r = P.poly_add(r, P.poly_scale(z_poly, s_ident))
    r = P.poly_add(r, P.poly_scale(Pp["s_sigma_4"], (-s_copy) % R_MOD))
    r = P.poly_add(r, P.poly_scale(z_poly, l1_z * alpha % R_MOD * alpha % R_MOD))
    z_n = pow(z_ch, size, R_MOD)
    quot = t_polys[0]
    for j in (1, 2, 3):
        quot = P.poly_add(quot, P.poly_scale(t_polys[j], pow(z_n, j, R_MOD)))
    return P.poly_add(r, P.poly_scale(quot, (-domain.evaluate_vanishing_polynomial(z_ch)) % R_MOD))


def forge_proof(pd: P.ProverData, comp: P.Composer, rng: P.StdRng) -> bytes:
    """forge_proof (proof.rs:1332-1682): a proof whose permutation argument and quotient are random, made to pass
    the V1 equation by solving q_arith_eval after z is known."""
    size = pd.size
    domain = P.EvaluationDomain(size)
    ck = pd.commit_key
    t = base_transcript(pd.label, pd.constraints, pd.comms, 1)
    public_inputs = comp.public_inputs_vec()
    dense_pi = [0] * size
    for i, v in zip(comp.public_input_indexes(), public_inputs):
        dense_pi[i] = v
    for pi in public_inputs:
        t.append_scalar(b"pi", pi)
    # round 1: honest wires
    wires = [[0] * size for _ in range(4)]
    for i, gt in enumerate(comp.constraints):
        for j, w in enumerate((gt.a, gt.b, gt.c, gt.d)):
            wires[j][i] = comp.witnesses[w]
    w_polys = [P.blind_poly(domain, wires[j], [P.fr_random(rng) for _ in range(2)]) for j in range(4)]
    for lab, p in zip((b"a_comm", b"b_comm", b"c_comm", b"d_comm"), w_polys):
        t.append_commitment(lab, P.commit(ck, p))
    # round 2: a random permutation polynomial
    beta = t.challenge_scalar(b"beta")
    t.append_scalar(b"beta", beta)
    gamma = t.challenge_scalar(b"gamma")
    z_poly = P.blind_poly(domain, [P.fr_random(rng) for _ in range(size)], [P.fr_random(rng) for _ in range(3)])
    z_comm = P.commit(ck, z_poly)
    t.append_commitment(b"z_comm", z_comm)
    # round 3: random linear quotient chunks
    ch = dict(alpha=t.challenge_scalar(b"alpha"), beta=beta, gamma=gamma)
    ch["range"] = t.challenge_scalar(b"range separation challenge")
    ch["logic"] = t.challenge_scalar(b"logic separation challenge")
    ch["fixed"] = t.challenge_scalar(b"fixed base separation challenge")
    ch["var"] = t.challenge_scalar(b"variable base separation challenge")
    t_polys = []
    for _ in range(4):
        c0, c1 = P.fr_random(rng), P.fr_random(rng)
        while c1 == 0:
            c1 = P.fr_random(rng)
        t_polys.append([c0, c1])
    t_comms = [P.commit(ck, p) for p in t_polys]
    for lab, cm in zip((b"t_low_comm", b"t_mid_comm", b"t_high_comm", b"t_fourth_comm"), t_comms):
        t.append_commitment(lab, cm)
    # round 4: honest evaluations, then q_arith_eval solved
    z_ch = t.challenge_scalar(b"z_challenge")
    zw = z_ch * domain.group_gen % R_MOD
    e = {}
    e["a"], e["b"], e["c"], e["d"] = (P.poly_eval(p, z_ch) for p in w_polys)
    e["s1"], e["s2"], e["s3"] = (P.poly_eval(pd.polys[f"s_sigma_{j}"], z_ch) for j in (1, 2, 3))
    e["z"] = P.poly_eval(z_poly, zw)
    for lab, k in ((b"a_eval", "a"), (b"b_eval", "b"), (b"c_eval", "c"), (b"d_eval", "d"), (b"s_sigma_1_eval", "s1"),
                   (b"s_sigma_2_eval", "s2"), (b"s_sigma_3_eval", "s3"), (b"z_eval", "z")):
        t.append_scalar(lab, e[k])
    e["a_w"], e["b_w"], e["d_w"] = P.poly_eval(w_polys[0], zw), P.poly_eval(w_polys[1], zw), P.poly_eval(w_polys[3], zw)
    e["q_c"], e["q_l"], e["q_r"] = (P.poly_eval(pd.polys[k], z_ch) for k in ("q_c", "q_l", "q_r"))
    for lab, k in ((b"a_w_eval", "a_w"), (b"b_w_eval", "b_w"), (b"d_w_eval", "d_w")):
        t.append_scalar(lab, e[k])
    alpha = ch["alpha"]
    z_h = domain.evaluate_vanishing_polynomial(z_ch)
    l1 = z_h * P.fr_inv(size * (z_ch - 1) % R_MOD) % R_MOD
    pi_eval = P.compute_barycentric_eval(dense_pi, z_ch, domain)
    r0 = (pi_eval - l1 * alpha * alpha
          - alpha * (e["a"] + beta * e["s1"] + gamma) * (e["b"] + beta * e["s2"] + gamma) % R_MOD
          * (e["c"] + beta * e["s3"] + gamma) % R_MOD * (e["d"] + gamma) % R_MOD * e["z"]) % R_MOD
    r_q0 = P.poly_eval(linearisation_poly(pd, ch, dict(e, q_arith=0), z_ch, z_poly, t_polys, dense_pi), z_ch)
    arith_base = (e["a"] * e["b"] * P.poly_eval(pd.polys["q_m"], z_ch) + e["a"] * P.poly_eval(pd.polys["q_l"], z_ch)
                  + e["b"] * P.poly_eval(pd.polys["q_r"], z_ch) + e["c"] * P.poly_eval(pd.polys["q_o"], z_ch)
                  + e["d"] * P.poly_eval(pd.polys["q_f"], z_ch) + P.poly_eval(pd.polys["q_c"], z_ch)) % R_MOD
    e["q_arith"] = (-r0 + pi_eval - r_q0) * P.fr_inv(arith_base) % R_MOD
    for lab, k in ((b"q_arith_eval", "q_arith"), (b"q_c_eval", "q_c"), (b"q_l_eval", "q_l"), (b"q_r_eval", "q_r")):
        t.append_scalar(lab, e[k])
    # round 5: the legacy opening
    v_ch = t.challenge_scalar(b"v_challenge")
    r_poly = linearisation_poly(pd, ch, e, z_ch, z_poly, t_polys, dense_pi)
    w_z = aggregate_witness([r_poly, *w_polys, *(pd.polys[f"s_sigma_{j}"] for j in (1, 2, 3))], z_ch, v_ch)
    v_w = t.challenge_scalar(b"v_w_challenge")
    w_zw = aggregate_witness([z_poly, w_polys[0], w_polys[1], w_polys[3]], zw, v_w)
    out = b"".join(P.g1_compress(c) for c in (*(P.commit(ck, p) for p in w_polys), z_comm, *t_comms, P.commit(ck, w_z), P.commit(ck, w_zw)))
    for k in OV.EVAL_ORDER:
        out += P.fr_to_bytes(e[k])
    assert len(out) == 1008
    return out
