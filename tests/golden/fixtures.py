"""Loaders for the committed fixtures (tests/golden/*.json)."""
import json
import os

from oracle import gg20_oracle as o

HERE = os.path.dirname(os.path.abspath(__file__))


def load_keyset(index: int = 0):
    """-> list of oracle.LocalKey for the 3 parties of key set `index`."""
    with open(os.path.join(HERE, "keys_t1n3.json")) as f:
        return _local_keys(json.load(f)["keysets"][index])


def edge_keysets_raw():
    """the key sets of keys_edge.json as stored (hex strings, with each row's shape and p~, q~, xhi)"""
    with open(os.path.join(HERE, "keys_edge.json")) as f:
        return json.load(f)["keysets"]


def load_edge_keysets():
    """-> one list of oracle.LocalKey per key set of keys_edge.json (keys at the edges of the accepted domain)"""
    return [_local_keys(ks) for ks in edge_keysets_raw()]


def _local_keys(ks):
    parties = ks["parties"]
    eks, stmts, pks = [], [], []
    for p in parties:
        n = int(p["p"], 16) * int(p["q"], 16)
        eks.append(o.EncryptionKey(n, n * n))
        stmts.append(o.DLogStatement(int(p["n_tilde"], 16), int(p["h1"], 16), int(p["h2"], 16)))
        pks.append(o.pt_mul(o.G, int(p["x_i"], 16)))
    y = o.pt_mul(o.G, int(ks["secret"], 16))
    keys = [o.LocalKey(i=p["i"], t=ks["t"], n=ks["n"], x_i=int(p["x_i"], 16),
                       dk=o.DecryptionKey(int(p["p"], 16), int(p["q"], 16)), pk_vec=pks, paillier_key_vec=eks,
                       h1_h2_n_tilde_vec=stmts, y_sum_s=y) for p in parties]
    return keys


def n_keysets() -> int:
    with open(os.path.join(HERE, "keys_t1n3.json")) as f:
        return len(json.load(f)["keysets"])


def load_all_keysets():
    return [load_keyset(i) for i in range(n_keysets())]
