"""Wire / on-disk formats of the reference (SURVEY.md section 8(f) rank 2): serde-JSON of the structs the GG20 protocol sends
and stores, written from and read into the engine's limb arrays, so that proofs and messages produced by the GPU engine can be
handed to the reference's own `verify` functions (bindings/rust/tests/reference_accepts_gpu_proofs.rs) and reference-generated
`local-share*.json` files can be loaded into `gg20.KeySets`.

Struct layouts (field names and order) are those of the in-tree `#[derive(Serialize, Deserialize)]` definitions:
  AliceProof {z,e,s,s1,s2}                       /root/reference/src/utilities/mta/range_proofs.rs:94-101
  MessageA {c, range_proofs}, MessageB {c, b_proof, beta_tag_proof}      src/utilities/mta/mod.rs:34-46
  PDLwSlackProof {z,u1,u2,u3,s1,s2,s3}, PDLwSlackStatement               src/utilities/zk_pdl_with_slack/mod.rs:40-66
  LocalKey {paillier_dk, pk_vec, keys_linear, paillier_key_vec, y_sum_s, h1_h2_n_tilde_vec, vss_scheme, i, t, n}
                                                 src/protocols/multi_party_ecdsa/gg_2020/state_machine/keygen/rounds.rs:309-322
  KeyGenBroadcastMessage1, KeyGenDecommitMessage1, SharedKeys, SignatureRecid      gg_2020/party_i.rs:96-135
The LEAF encodings live in crates that are not vendored (curv-kzen 0.9, kzen-paillier 0.4.2, zk-paillier 0.4.3) and are
RECALLED [R], not verified in this container — they are isolated in `Encoding` so that one run of the Rust test pins (or
corrects) them in one place:
  BigInt      -> lower-case hex string of `to_bytes()` (human-readable serializers), "0" -> "00" [R]
  Scalar<E>   -> {"curve": "secp256k1", "scalar": <32 bytes>}                                 [R]
  Point<E>    -> {"curve": "secp256k1", "point": <33 bytes, SEC1 compressed>}                  [R]
     bytes: hex string (`Encoding.bytes_as="hex"`, curv 0.9 with human-readable formats) or array of numbers ("array", serde's
     default for Vec<u8> in JSON)                                                             [R]
  EncryptionKey -> {"n": BigInt}; DecryptionKey -> {"p": BigInt, "q": BigInt}                  [R] (kzen-paillier minimal keys)
  DLogStatement -> {"N","g","ni"}; NiCorrectKeyProof -> {"sigma_vec": [...]}; CompositeDLogProof -> {"x","y"}   [R]
  DLogProof -> {"pk","pk_t_rand_commitment","challenge_response"}                             [R]
  VerifiableSS -> {"parameters": {"threshold","share_count"}, "commitments": [Point]}         [R]
No arithmetic happens here (the 33-byte point encodings come from the engine's `Point::to_bytes(true)` entry point when an
engine is supplied, else from the parity bit of y)."""
from __future__ import annotations

import json
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

Point = Optional[Tuple[int, int]]
CURVE = "secp256k1"


@dataclass
class Encoding:
    bytes_as: str = "hex"          # "hex" | "array"   [R]

    def bigint(self, x: int) -> str:
        x = int(x)
        if x < 0:
            raise ValueError("negative BigInt on the wire")
        return x.to_bytes(max(1, (x.bit_length() + 7) // 8), "big").hex()

    def bigint_from(self, s: Any) -> int:
        if isinstance(s, str):
            return int(s, 16) if s else 0
        return int.from_bytes(bytes(s), "big")

    def raw(self, b: bytes) -> Any:
        return b.hex() if self.bytes_as == "hex" else list(b)

    def raw_from(self, v: Any) -> bytes:
        return bytes.fromhex(v) if isinstance(v, str) else bytes(v)

    def scalar(self, x: int) -> Dict[str, Any]:
        return {"curve": CURVE, "scalar": self.raw(int(x).to_bytes(32, "big"))}

    def scalar_from(self, d: Dict[str, Any]) -> int:
        assert d["curve"] == CURVE
        return int.from_bytes(self.raw_from(d["scalar"]), "big")

    def point(self, p: Point) -> Dict[str, Any]:
        if p is None:
            return {"curve": CURVE, "point": self.raw(b"\x00")}
        return {"curve": CURVE, "point": self.raw(bytes([2 + (p[1] & 1)]) + p[0].to_bytes(32, "big"))}

    def point_from(self, d: Dict[str, Any], decompress) -> Point:
        assert d["curve"] == CURVE
        b = self.raw_from(d["point"])
        return None if b == b"\x00" else decompress(b)


DEFAULT = Encoding()


# ------------------------------------------------------------------------------------------------- proofs and messages
def alice_proof(pf: Dict[str, int], enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """pf = {"z","e","s","s1","s2"} as returned by gg20.alice_proof_generate (one proof)"""
    return {k: enc.bigint(pf[k]) for k in ("z", "e", "s", "s1", "s2")}


def dlog_proof(row40, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """row40 = one row of gg20.dlog_prove: pk 16 | pk_t_rand_commitment 16 | challenge_response 8 (uint32 limbs)"""
    def pt(limbs):
        v = int.from_bytes(limbs.tobytes(), "little")
        return None if v == 0 else (v & ((1 << 256) - 1), v >> 256)
    return {"pk": enc.point(pt(row40[:16])), "pk_t_rand_commitment": enc.point(pt(row40[16:32])),
            "challenge_response": enc.scalar(int.from_bytes(row40[32:40].tobytes(), "little"))}


def message_a(c: int, proofs: Sequence[Dict[str, int]], enc: Encoding = DEFAULT) -> Dict[str, Any]:
    return {"c": enc.bigint(c), "range_proofs": [alice_proof(p, enc) for p in proofs]}


def message_b(c: int, b_proof_row, beta_tag_proof_row, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    return {"c": enc.bigint(c), "b_proof": dlog_proof(b_proof_row, enc), "beta_tag_proof": dlog_proof(beta_tag_proof_row, enc)}


def pdl_proof(pf: Dict[str, Any], enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """pf = {"z","u1" (point),"u2","u3","s1","s2","s3"}"""
    return {"z": enc.bigint(pf["z"]), "u1": enc.point(pf["u1"]), "u2": enc.bigint(pf["u2"]), "u3": enc.bigint(pf["u3"]),
            "s1": enc.bigint(pf["s1"]), "s2": enc.bigint(pf["s2"]), "s3": enc.bigint(pf["s3"])}


def pdl_statement(ciphertext: int, n: int, Q: Point, G: Point, h1: int, h2: int, n_tilde: int, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    return {"ciphertext": enc.bigint(ciphertext), "ek": encryption_key(n, enc), "Q": enc.point(Q), "G": enc.point(G),
            "h1": enc.bigint(h1), "h2": enc.bigint(h2), "N_tilde": enc.bigint(n_tilde)}


def encryption_key(n: int, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    return {"n": enc.bigint(n)}


def dlog_statement(N: int, g: int, ni: int, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    return {"N": enc.bigint(N), "g": enc.bigint(g), "ni": enc.bigint(ni)}


def signature_recid(r: int, s: int, recid: int, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """`SignatureRecid {r, s, recid}` (gg_2020/party_i.rs:130-135)"""
    return {"r": enc.scalar(r), "s": enc.scalar(s), "recid": int(recid)}


def keygen_broadcast1(n: int, stmt: Tuple[int, int, int], com: int, sigma_vec: Sequence[int], proof_h1: Tuple[int, int], proof_h2: Tuple[int, int],
                      enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """`KeyGenBroadcastMessage1` (gg_2020/party_i.rs:96-104)"""
    return {"e": encryption_key(n, enc), "dlog_statement": dlog_statement(*stmt, enc), "com": enc.bigint(com),
            "correct_key_proof": {"sigma_vec": [enc.bigint(s) for s in sigma_vec]},
            "composite_dlog_proof_base_h1": {"x": enc.bigint(proof_h1[0]), "y": enc.bigint(proof_h1[1])},
            "composite_dlog_proof_base_h2": {"x": enc.bigint(proof_h2[0]), "y": enc.bigint(proof_h2[1])}}


# ------------------------------------------------------------------------------------------------- offline-stage round messages
def _row_pt(limbs) -> Point:
    v = int.from_bytes(limbs.tobytes(), "little")
    return None if v == 0 else (v & ((1 << 256) - 1), v >> 256)


def _row_int(limbs) -> int:
    return int.from_bytes(limbs.tobytes(), "little")


def pedersen_proof(row64, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """curv `PedersenProof {e, a1, a2, com, z1, z2}` [R] from one row of gg20.pedersen_prove (e 8 | a1 16 | a2 16 | z1 8 | z2 8) and its
    commitment; `com` is filled by the caller (it is T_i)"""
    return {"e": enc.scalar(_row_int(row64[:8])), "a1": enc.point(_row_pt(row64[8:24])), "a2": enc.point(_row_pt(row64[24:40])), "com": None,
            "z1": enc.scalar(_row_int(row64[40:48])), "z2": enc.scalar(_row_int(row64[48:56]))}


def heg_proof(row48, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """curv `HomoELGamalProof {T, A3, z1, z2}` [R] from one row of gg20.heg_prove (T 16 | A3 16 | z1 8 | z2 8)"""
    return {"T": enc.point(_row_pt(row48[:16])), "A3": enc.point(_row_pt(row48[16:32])), "z1": enc.scalar(_row_int(row48[32:40])),
            "z2": enc.scalar(_row_int(row48[40:48]))}


def sign_broadcast_phase1(com: int, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """`SignBroadcastPhase1 {com}` (gg_2020/party_i.rs:113-116)"""
    return {"com": enc.bigint(com)}


def sign_decommit_phase1(blind_factor: int, g_gamma_i: Point, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """`SignDecommitPhase1 {blind_factor, g_gamma_i}` (gg_2020/party_i.rs:118-122)"""
    return {"blind_factor": enc.bigint(blind_factor), "g_gamma_i": enc.point(g_gamma_i)}


def offline_message(kind: str, body: Any) -> Dict[str, Any]:
    """`OfflineProtocolMessage(OfflineM::<kind>(body))` (state_machine/sign.rs:478-490): a newtype around an externally tagged enum;
    tuple bodies are JSON arrays, the newtype wrappers GammaI / WI / DeltaI / TI / TIProof / RDash / SI / HEGProof (sign/rounds.rs:33-49)
    are transparent"""
    assert kind in ("M1", "M2", "M3", "M4", "M5", "M6")
    return {kind: body}


def msg(sender: int, receiver: Optional[int], body: Any) -> Dict[str, Any]:
    """round_based `Msg {sender, receiver, body}` [R] (1-based party indices; receiver = null for a broadcast)"""
    return {"sender": int(sender), "receiver": None if receiver is None else int(receiver), "body": body}


# ------------------------------------------------------------------------------------------------- LocalKey (local-share*.json)
def local_key(lk, commitments: Sequence[Point], enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """`LocalKey<Secp256k1>` from an object with the fields of oracle.LocalKey (i, t, n, x_i, dk.p, dk.q, pk_vec,
    paillier_key_vec[*].n, h1_h2_n_tilde_vec[*].(N,g,ni), y_sum_s); `commitments` = the summed Feldman commitments"""
    return {
        "paillier_dk": {"p": enc.bigint(lk.dk.p), "q": enc.bigint(lk.dk.q)},
        "pk_vec": [enc.point(p) for p in lk.pk_vec],
        "keys_linear": {"y": enc.point(lk.pk_vec[lk.i - 1]), "x_i": enc.scalar(lk.x_i)},
        "paillier_key_vec": [encryption_key(ek.n, enc) for ek in lk.paillier_key_vec],
        "y_sum_s": enc.point(lk.y_sum_s),
        "h1_h2_n_tilde_vec": [dlog_statement(st.N, st.g, st.ni, enc) for st in lk.h1_h2_n_tilde_vec],
        "vss_scheme": {"parameters": {"threshold": lk.t, "share_count": lk.n}, "commitments": [enc.point(p) for p in commitments]},
        "i": lk.i, "t": lk.t, "n": lk.n,
    }


@dataclass
class DecryptionKey:
    """paillier `DecryptionKey` {p, q}"""
    p: int
    q: int


@dataclass
class EncryptionKey:
    """paillier `EncryptionKey` {n, nn}"""
    n: int
    nn: Optional[int] = None        # the engine derives N^2 on the device


@dataclass
class DLogStatement:
    """zk-paillier `DLogStatement` {N, g, ni} = (N~, h1, h2)"""
    N: int
    g: int
    ni: int


@dataclass
class LoadedLocalKey:
    """What gg20.KeySets needs from a `LocalKey` (duck-typed like oracle.LocalKey)"""
    i: int
    t: int
    n: int
    x_i: int
    dk: DecryptionKey
    pk_vec: List[Point]
    paillier_key_vec: List[EncryptionKey]
    h1_h2_n_tilde_vec: List[DLogStatement]
    y_sum_s: Point
    vss_commitments: List[Point]


def load_local_key(doc: Dict[str, Any], decompress, enc: Encoding = DEFAULT) -> LoadedLocalKey:
    """Parse a reference `local-share*.json` document (examples/gg20_keygen.rs:52-55).  `decompress(bytes33) -> (x, y)` is the
    engine's `Point::from_bytes` (Engine.point_decompress) or any equivalent."""
    B = enc.bigint_from
    pt = lambda d: enc.point_from(d, decompress)
    return LoadedLocalKey(
        i=int(doc["i"]), t=int(doc["t"]), n=int(doc["n"]), x_i=enc.scalar_from(doc["keys_linear"]["x_i"]),
        dk=DecryptionKey(B(doc["paillier_dk"]["p"]), B(doc["paillier_dk"]["q"])),
        pk_vec=[pt(p) for p in doc["pk_vec"]],
        paillier_key_vec=[EncryptionKey(B(e["n"])) for e in doc["paillier_key_vec"]],
        h1_h2_n_tilde_vec=[DLogStatement(B(s["N"]), B(s["g"]), B(s["ni"])) for s in doc["h1_h2_n_tilde_vec"]],
        y_sum_s=pt(doc["y_sum_s"]), vss_commitments=[pt(p) for p in doc["vss_scheme"]["commitments"]])


def parse_offline_message(m: Dict[str, Any], decompress, enc: Encoding = DEFAULT) -> Dict[str, Any]:
    """Inverse of msg(...offline_message(...)): a `Msg<OfflineProtocolMessage>` document from a peer -> {"sender", "receiver", "kind"} plus
    the decoded fields in the shapes the batch calls take (integers, (x, y) points, proof dicts / 40-limb DLogProof rows as integers):
      M1: c, range_proofs [{z,e,s,s1,s2}], com          M2: gamma / w = {c, b_proof, beta_tag_proof} with proofs as {pk, pk_t_rand_commitment,
      M3: delta, T, pedersen {e,a1,a2,com,z1,z2}              challenge_response}
      M4: blind_factor, g_gamma                          M5: R_dash, pdl [{z,u1,u2,u3,s1,s2,s3}]          M6: S, heg {T,A3,z1,z2}
    Field widths are NOT checked here: the verify-side wrappers (gg20._Screen) reject over-wide values per element."""
    B, S = enc.bigint_from, enc.scalar_from
    P = lambda d: enc.point_from(d, decompress)
    (kind, body), = m["body"].items()
    out = {"sender": int(m["sender"]), "receiver": None if m["receiver"] is None else int(m["receiver"]), "kind": kind}
    dl = lambda d: {"pk": P(d["pk"]), "pk_t_rand_commitment": P(d["pk_t_rand_commitment"]), "challenge_response": S(d["challenge_response"])}
    mb = lambda d: {"c": B(d["c"]), "b_proof": dl(d["b_proof"]), "beta_tag_proof": dl(d["beta_tag_proof"])}
    if kind == "M1":
        out.update(c=B(body[0]["c"]), range_proofs=[{k: B(pf[k]) for k in ("z", "e", "s", "s1", "s2")} for pf in body[0]["range_proofs"]], com=B(body[1]["com"]))
    elif kind == "M2":
        out.update(gamma=mb(body[0]), w=mb(body[1]))
    elif kind == "M3":
        pf = body[2]
        out.update(delta=S(body[0]), T=P(body[1]), pedersen={"e": S(pf["e"]), "a1": P(pf["a1"]), "a2": P(pf["a2"]), "com": P(pf["com"]), "z1": S(pf["z1"]), "z2": S(pf["z2"])})
    elif kind == "M4":
        out.update(blind_factor=B(body["blind_factor"]), g_gamma=P(body["g_gamma_i"]))
    elif kind == "M5":
        out.update(R_dash=P(body[0]), pdl=[{"z": B(pf["z"]), "u1": P(pf["u1"]), "u2": B(pf["u2"]), "u3": B(pf["u3"]), "s1": B(pf["s1"]), "s2": B(pf["s2"]), "s3": B(pf["s3"])}
                                            for pf in body[1]])
    elif kind == "M6":
        pf = body[1]
        out.update(S=P(body[0]), heg={"T": P(pf["T"]), "A3": P(pf["A3"]), "z1": S(pf["z1"]), "z2": S(pf["z2"])})
    else:
        raise ValueError("unknown OfflineM variant " + kind)
    return out


def dumps(doc: Any) -> str:
    """serde_json's compact form"""
    return json.dumps(doc, separators=(",", ":"))
