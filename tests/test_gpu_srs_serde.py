"""GPU: G1 decode / encode of params file points (zkb_g1_decode / zkb_g1_encode) and ParamsKZG.read_custom / write_custom in every
SerdeFormat.  The compressed encoding is pinned by the reference fixture's own vk and proof points; every decoded point is checked
against the big-integer oracle (oracle/pyref.py)."""
import os
import re

import numpy as np
import pytest

import pyref as P

pytestmark = pytest.mark.gpu

Q = P.Q_MOD
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = eval(re.search(r"#define ZKB_SERDE_CHUNK_POINTS (.+)", open(os.path.join(ROOT, "include", "zkb200.h")).read()).group(1).replace("u", ""))


def aff(pt):
    return np.zeros(8, dtype=np.uint64) if pt is None else np.array(P.limbs(P.to_mont(pt[0], Q)) + P.limbs(P.to_mont(pt[1], Q)), dtype=np.uint64)


def pt_of(row):
    row = np.asarray(row).view(np.uint64)
    if not row.any():
        return None
    return (P.from_mont(P.from_limbs(row[:4]), Q), P.from_mont(P.from_limbs(row[4:]), Q))


def host(t):
    return t if isinstance(t, np.ndarray) else t.cpu().numpy().view(np.uint64 if t.dtype.itemsize == 8 else np.uint8)


def decode(fmt, src, n, in_dev=False, out_dev=False):
    import torch
    from zkb200.params import g1_decode
    src = torch.from_numpy(src).cuda() if in_dev else src
    out = torch.empty((n, 8), dtype=torch.int64, device="cuda") if out_dev else np.empty((n, 8), dtype=np.uint64)
    rep = g1_decode(fmt, src, n, out)
    return host(out).reshape(n, 8), rep


def encode(fmt, pts, in_dev=False, out_dev=False):
    import torch
    from zkb200.params import SerdeFormat, g1_encode
    n = pts.shape[0]
    nb = n * SerdeFormat(fmt).g1_len
    src = torch.from_numpy(pts.view(np.int64)).cuda() if in_dev else pts
    out = torch.empty(nb, dtype=torch.uint8, device="cuda") if out_dev else np.empty(nb, dtype=np.uint8)
    g1_encode(fmt, src, out)
    return host(out)


@pytest.fixture(scope="module")
def points():
    """the g and g_lagrange of unsafe_setup_with_s at k = 10, as one host array of 2048 points"""
    from zkb200.params import ParamsKZG
    p = ParamsKZG.unsafe_setup_with_s(10, 4321)
    return np.concatenate([host(p.g), host(p.g_lagrange)])


def tiled(points, n):
    return np.ascontiguousarray(np.resize(points, (n, 8)))


def test_fixture_points_decode_and_encode(golden):
    """the 7 vk points and the 11 proof points of the reference fixture decode to exactly pyref.g1_decompress, and encode back"""
    from zkb200.params import SerdeFormat as SF
    vk, proof = bytes.fromhex(golden["vk_hex"]), bytes.fromhex(golden["proof_hex"])
    nw = sum(golden["num_witness"]) + golden["quotient_num_chunk"]
    enc = [vk[8 + 32 * i: 40 + 32 * i] for i in range(7)] + [proof[32 * i: 32 * i + 32] for i in list(range(nw)) + [26, 27]]
    assert len(enc) == 18
    src = np.frombuffer(b"".join(enc), dtype=np.uint8).copy()
    for in_dev, out_dev in ((False, False), (True, True)):
        out, rep = decode(SF.Processed, src, 18, in_dev, out_dev)
        assert rep.count == 0 and rep.first_bad is None
        assert [pt_of(r) for r in out] == [P.g1_decompress(e) for e in enc]
        for i, pp in enumerate(golden["preprocessed"]):
            assert (out[i] == np.array(pp["x"] + pp["y"], dtype=np.uint64)).all()
        assert encode(SF.Processed, out, in_dev, out_dev).tobytes() == src.tobytes()


def test_random_points_encode_and_roundtrip(points):
    from zkb200.params import SerdeFormat as SF
    enc = encode(SF.Processed, points, in_dev=True)
    assert [enc[32 * i: 32 * i + 32].tobytes() for i in range(len(points))] == [P.g1_compress(pt_of(r)) for r in points]
    for fmt in (SF.Processed, SF.RawBytes, SF.RawBytesUnchecked):
        e = encode(fmt, points)
        assert e.nbytes == len(points) * fmt.g1_len
        for in_dev, out_dev in ((False, False), (False, True), (True, False), (True, True)):
            out, rep = decode(fmt, e, len(points), in_dev, out_dev)
            assert rep.count == 0 and (out == points).all(), (fmt, in_dev, out_dev)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, CHUNK - 1, CHUNK, CHUNK + 1])
def test_streaming_sizes(points, n):
    """host streaming path at every chunk edge: host and device paths give identical bytes, both the identity on decode(encode)"""
    from zkb200.params import SerdeFormat as SF
    pts = tiled(points, n)
    for fmt in (SF.Processed, SF.RawBytes):
        e_host = encode(fmt, pts)
        e_dev = encode(fmt, pts, True, True)
        assert e_host.tobytes() == e_dev.tobytes()
        d_host, r1 = decode(fmt, e_host, n)
        d_dev, r2 = decode(fmt, e_host, n, True, True)
        assert r1 == r2 and r1.count == 0
        assert d_host.tobytes() == d_dev.tobytes() == pts.tobytes()


def _q_limbs_bytes(v):
    return v.to_bytes(32, "little")


def test_injected_faults_processed(points):
    """exact first index, count and reason; a flipped sign bit is the negated point, the identity is accepted"""
    from zkb200.params import SerdeFormat as SF
    n = CHUNK + 100                                        # faults on both sides of a chunk boundary of the host path
    pts = tiled(points, n)
    enc = encode(SF.Processed, pts, in_dev=True).reshape(n, 32).copy()
    x_bad = 1
    while P.fq_sqrt((x_bad ** 3 + 3) % Q) is not None:
        x_bad += 1
    faults = {CHUNK + 7: 1, 5000: 2, 40: 3, CHUNK - 1: 3, 777: 1}
    for i, reason in faults.items():
        if reason == 1:
            enc[i, 31] |= 0x80
        elif reason == 2:
            enc[i] = np.frombuffer(_q_limbs_bytes(Q + 5), dtype=np.uint8)
        else:
            enc[i] = np.frombuffer(_q_limbs_bytes(x_bad), dtype=np.uint8)
    flipped, ident = [3, CHUNK + 50], [10, CHUNK + 1]
    for i in flipped:
        enc[i, 31] ^= 0x40
    for i in ident:
        enc[i] = 0
    want = pts.copy()
    for i in flipped:
        want[i] = aff(P.g1_neg(pt_of(pts[i])))
    for i in ident + list(faults):
        want[i] = 0
    flat = enc.reshape(-1)
    for in_dev, out_dev in ((False, False), (True, True), (False, True)):
        for _ in range(2):                                 # same report on every run
            out, rep = decode(SF.Processed, flat, n, in_dev, out_dev)
            assert rep == (40, len(faults), 3)
            assert (out == want).all()
    # the first bad point alone decides the reason
    enc2 = encode(SF.Processed, tiled(points, 64)).reshape(64, 32).copy()
    enc2[9, 31] |= 0x80
    enc2[30] = np.frombuffer(_q_limbs_bytes(x_bad), dtype=np.uint8)
    assert decode(SF.Processed, enc2.reshape(-1), 64)[1] == (9, 2, 1)


def test_injected_faults_raw(points):
    from zkb200.params import SerdeFormat as SF
    n = CHUNK + 100
    pts = tiled(points, n)
    bad = pts.copy()
    q_top = Q >> 192
    bad[12, 3] = np.uint64(q_top + 1)                   # x >= q
    bad[CHUNK + 3, 7] = np.uint64(0xFFFFFFFFFFFFFFFF)   # y >= q
    bad[600, 4] ^= np.uint64(1)                         # off the curve
    bad[CHUNK + 90] = 0                                 # the identity
    want = pts.copy()
    want[[12, CHUNK + 3, 600, CHUNK + 90]] = 0
    for in_dev, out_dev in ((False, False), (True, True), (True, False)):
        out, rep = decode(SF.RawBytes, bad.view(np.uint8).reshape(-1), n, in_dev, out_dev)
        assert rep == (12, 3, 2)
        assert (out == want).all()
    out, rep = decode(SF.RawBytesUnchecked, bad.view(np.uint8).reshape(-1), n)
    assert rep.count == 0 and (out == bad).all()
    bad[12] = pts[12]
    assert decode(SF.RawBytes, bad.view(np.uint8).reshape(-1), n)[1] == (600, 2, 3)


def _params_with_g2(k):
    import pairing_ref as PR
    from test_srs_serde_cpu import raw_g2
    from zkb200.params import PARAMS_G2_SECRET_POWER, ParamsKZG
    p = ParamsKZG.unsafe_setup_with_s(k, 4321 + k)
    p.g2, p.s_g2 = raw_g2(PR.G2), np.array(PARAMS_G2_SECRET_POWER, dtype=np.uint64).tobytes()
    return p


@pytest.mark.parametrize("k", list(range(1, 13)) + [20])
def test_params_file_every_format_pair(tmp_path, k):
    """write(a) -> read(a) -> write(b) -> read(b) for every pair of formats: sizes are expected_file_len, arrays come back exactly"""
    from zkb200.params import ParamsKZG, SerdeFormat as SF
    p = _params_with_g2(k)
    g, gl = host(p.g), host(p.g_lagrange)
    for a in SF:
        pa = tmp_path / f"a{int(a)}"
        p.write_custom(str(pa), a)
        assert pa.stat().st_size == ParamsKZG.expected_file_len(k, a)
        qa = ParamsKZG.read_custom(str(pa), a, to_device=(a != SF.RawBytes))
        for b in SF:
            pb = tmp_path / f"b{int(b)}"
            qa.write_custom(str(pb), b)
            assert pb.stat().st_size == ParamsKZG.expected_file_len(k, b)
            for to_device in (True, False):
                qb = ParamsKZG.read_custom(str(pb), b, to_device=to_device)
                assert qb.k == k and (host(qb.g) == g).all() and (host(qb.g_lagrange) == gl).all(), (a, b, to_device)
                assert qb.g2 == p.g2 and qb.s_g2 == p.s_g2
            qb.check_s_g2()


def test_params_file_corrupted_point_names_array_and_index(tmp_path):
    from zkb200.params import ParamsKZG, SerdeFormat as SF
    k = 6
    n = 1 << k
    p = _params_with_g2(k)
    for fmt in (SF.Processed, SF.RawBytes):
        path = tmp_path / f"p{int(fmt)}"
        p.write_custom(str(path), fmt)
        good = path.read_bytes()
        g1 = fmt.g1_len
        for off, msg in ((4 + n * g1 + 5 * g1, r"g_lagrange\[5\] has (flag bit 7 set|a coordinate >= q); 2 bad point"),
                         (4 + 17 * g1, r"g\[17\] has (flag bit 7 set|a coordinate >= q); 2 bad point")):
            raw = bytearray(good)
            last = off + g1 - 1 if fmt is SF.Processed else off + 31   # Processed: the flag byte; raw: the top byte of x
            raw[last] |= 0x80
            raw[last + 3 * g1] |= 0x80                                  # a second bad point further on in the same array
            path.write_bytes(bytes(raw))
            with pytest.raises(ValueError, match=msg):
                ParamsKZG.read_custom(str(path), fmt)
        raw = bytearray(good)
        raw[4 + 2 * n * g1 + 2 * g1 - 1] |= 0x80                        # g2
        path.write_bytes(bytes(raw))
        with pytest.raises(ValueError, match=r"\bg2 has"):
            ParamsKZG.read_custom(str(path), fmt, to_device=False)
        path.write_bytes(good[:-7])
        with pytest.raises(ValueError, match="truncated at s_g2"):
            ParamsKZG.read_custom(str(path), fmt)
    # unchecked reads keep whatever the file holds
    path = tmp_path / "u"
    p.write_custom(str(path))
    raw = bytearray(path.read_bytes())
    raw[4 + 31] |= 0x80
    path.write_bytes(bytes(raw))
    q = ParamsKZG.read_custom(str(path), to_device=False)
    assert q.g[0, 3] >> np.uint64(56) == raw[4 + 31]


def test_proof_with_params_from_processed_file(tmp_path):
    """k = 13 SuperCircuit stand-in: the proof with params read back from a Processed file is byte-identical to the proof with the
    original params, and the oracle verifier accepts it"""
    import standins
    from test_gpu_standins import prove_gpu, verify_gpu_proof
    from zkb200.params import ParamsKZG, SerdeFormat as SF
    s = 4321
    params = ParamsKZG.unsafe_setup_with_s(13, s)
    path = tmp_path / "params13"
    params.write_custom(str(path), SF.Processed)
    back = ParamsKZG.read_custom(str(path), SF.Processed)
    sc = standins.super_shape(13, seed=13, advice=64, scale=1.0, n_gates=120)
    pk0, proof0, _, _, _ = prove_gpu(sc, params)
    pk1, proof1, fixed, sigma, inst = prove_gpu(sc, back)
    assert proof1 == proof0
    ok, rejected, checked = verify_gpu_proof(sc, pk1, proof1, inst, s, fixed, sigma)
    assert ok and rejected and checked == 2


def test_large_k22_host_and_device_paths(tmp_path):
    """2^22 points in each of g and g_lagrange: the host and device read paths agree byte for byte with the original arrays, and
    sampled points match the oracle's decompression"""
    from zkb200.params import ParamsKZG, SerdeFormat as SF
    k = 22
    p = ParamsKZG.unsafe_setup_with_s(k, 98765)
    g, gl = host(p.g), host(p.g_lagrange)
    path = tmp_path / "params22"
    p.write_custom(str(path), SF.Processed)
    assert path.stat().st_size == ParamsKZG.expected_file_len(k, SF.Processed)
    raw = path.read_bytes()
    dev = ParamsKZG.read_custom(str(path), SF.Processed, to_device=True)
    hst = ParamsKZG.read_custom(str(path), SF.Processed, to_device=False)
    assert host(dev.g).tobytes() == hst.g.tobytes() == g.tobytes()
    assert host(dev.g_lagrange).tobytes() == hst.g_lagrange.tobytes() == gl.tobytes()
    rng = np.random.default_rng(22)
    n = 1 << k
    for i in rng.integers(0, 2 * n, size=64).tolist() + [0, n - 1, n, 2 * n - 1]:
        row = hst.g[i] if i < n else hst.g_lagrange[i - n]
        assert pt_of(row) == P.g1_decompress(raw[4 + 32 * i: 36 + 32 * i])
