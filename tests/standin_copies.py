"""Copy constraints of the stand-in circuits (tests/standins.py), for the witness check.

A stand-in keeps only the sigma columns its permutations produce: permutation column j holds c_0[pi_j(r)] at usable row r (pi_0 =
identity).  The permutations are drawn from the stand-in's seeded torch generator after the lookup-pair row draws, so they are
replayed here with the same generator calls; `copies` checks the replay against sigma at a few cells.  The copy list is
(j, r) ~ (0, pi_j(r)) for j >= 1 and every usable row r: the same cycles as sigma.  Test / benchmark infrastructure."""
import numpy as np
import torch

R_MOD = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
ROOT_OF_UNITY_28 = 0x03DDB9F5166D18B798865EA93DD31F743215CF6DD39329C8D34F1ED960C37C9C
DELTA = pow(7, 1 << 28, R_MOD)


def permutations(sc):
    """[pi_0, ..., pi_{P-1}] of the stand-in, each a tensor of `usable` rows on the stand-in's device"""
    dev = sc.ops.device
    gen = torch.Generator(device=dev)
    gen.manual_seed(sc.seed)
    tables, width = sc.shape["lookup_tables"], sc.shape["lookup_width"]
    n_pairs = (sc.c_perm0 - sc.c_pair0) // width
    for pr in range(n_pairs):
        torch.randint(0, tables[pr // (n_pairs // len(tables))], (sc.n,), device=dev, generator=gen)
    return [torch.arange(sc.usable, device=dev)] + [torch.randperm(sc.usable, device=dev, generator=gen) for _ in range(sc.P - 1)]


def _canonical(mont_limbs):
    """Montgomery limbs -> the integer they stand for (x = m / 2^256 mod r)"""
    m = sum(int(v) << (64 * i) for i, v in enumerate(mont_limbs))
    return m * pow(1 << 256, -1, R_MOD) % R_MOD


def copies(sc, pis=None, spot=8):
    """the copy list as an int32 tensor (m, 4) on the stand-in's device: (j, r, 0, pi_j(r)) for j = 1 .. P-1, r < usable"""
    pis = pis or permutations(sc)
    dev, usable = sc.ops.device, sc.usable
    omega = pow(ROOT_OF_UNITY_28, 1 << (28 - sc.k), R_MOD)
    rng = np.random.default_rng(sc.seed)
    for j in range(sc.P):   # sigma_j[r] = delta^(j+1 mod P) * omega^(row of c_0[pi_j(r)] in column j+1 mod P)
        jn = (j + 1) % sc.P
        inv = torch.empty(usable, dtype=torch.int64, device=dev)
        inv[pis[jn]] = torch.arange(usable, device=dev)
        for r in rng.integers(0, usable, size=max(1, spot // sc.P + 1)):
            t = int(inv[pis[j][int(r)]])
            got = _canonical(sc.host(sc.sigma[j][int(r):int(r) + 1])[0])
            assert got == pow(DELTA, jn, R_MOD) * pow(omega, t, R_MOD) % R_MOD, "the permutation replay does not match sigma"
    rows = torch.arange(usable, device=dev, dtype=torch.int32)
    parts = [torch.stack([torch.full_like(rows, j), rows, torch.zeros_like(rows), pis[j].to(torch.int32)], dim=1) for j in range(1, sc.P)]
    return torch.cat(parts).contiguous() if parts else torch.zeros((0, 4), dtype=torch.int32, device=dev)


def witness(sc, challenges):
    """(fixed, advice, instances) tensors of the stand-in synthesised with the given challenge values (Montgomery uint64[4] each)"""
    adv = [None] * sc.cs.num_advice
    for phase in range(sc.cs.num_phases()):
        for c, t in sc.synthesize_dev(phase, {i: challenges[i] for i in range(len(challenges))}).items():
            adv[c] = t
    inst = []
    for t in sc.instances:
        col = torch.zeros((sc.n, 4), dtype=torch.int64, device=t.device)
        col[: t.shape[0]] = t
        inst.append(col)
    return list(sc.fixed), adv, inst
