"""CPU: the per-pixel fragment list of raster_forward_kernel does not depend on the order in which a tile lists its faces.

The two halves of a z-clipped quad exclude each other (the one nearer to the pixel stays), and a half only sees its other
half while that one is in the list: so which K fragments a pixel keeps depends on the order the candidates are offered in.
The oracle (oracle/raster_oracle.c, as PyTorch3D's CPU rasterizer) offers them in the clipped mesh's face order, where a
quad's halves are adjacent; the kernel lists slots in whatever order its warps win their atomics, and slot F + f holds the
second half of face f.  tests/host_math/dbw_fraglist_host.cpp compiles dbw_fraglist.cuh -- fraglist_offer and the ordering
step the kernel applies before offering (frag_order_rank / frag_order_slot) -- and these tests feed it random candidate sets
in many list orders: the list must always equal the oracle's queue."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import pt3d

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'host_math', 'dbw_fraglist_host.cpp')
RAW, SORTED, SCANNED = 0, 1, 2          # hm_list modes: list order as given / fast-path sort / chunked-path scan order


@pytest.fixture(scope='module')
def fl():
    out_dir = os.path.join(HERE, 'host_math', '_build')
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, 'libdbw_fraglist_host.so')
    gxx = '/usr/bin/g++' if os.path.exists('/usr/bin/g++') else 'g++'
    subprocess.run([gxx, '-O2', '-ffp-contract=off', '-std=c++17', '-fPIC', '-shared', '-Wall', '-Werror', '-Wno-unknown-pragmas', SRC, '-o', so], check=True)
    return ctypes.CDLL(so)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _kernel_list(fl, K, F, mode, cands):
    """cands: [(slot, pz, sd, neighbour slot)] in list order -> [(slot, sd)] the list keeps, front to back"""
    n = len(cands)
    slot = np.array([c[0] for c in cands], np.int32)
    pz = np.array([c[1] for c in cands], np.float32)
    sd = np.array([c[2] for c in cands], np.float32)
    nb = np.array([c[3] for c in cands], np.int32)
    out_slot, out_sd = np.zeros(K, np.int32), np.zeros(K, np.float32)
    cnt = fl.hm_list(K, F, n, mode, _p(pz), _p(slot), _p(sd), _p(nb), _p(out_slot), _p(out_sd))
    assert cnt >= 0, 'the ordering step lost or duplicated an entry'
    return [(int(s), float(d)) for s, d in zip(out_slot[:cnt], out_sd[:cnt])]


def _oracle_queue(K, cands):
    """the per-pixel queue of oracle/raster_oracle.c: candidates (depth, clipped face index, signed distance, clipped index of
    the other half or -1) offered in the order given; kept as the K smallest (depth, face, distance) tuples, ascending; a half
    of a z-clipped quad drops its other half from the queue if it is nearer to the pixel (|distance|), else is dropped"""
    q = []
    for z, f, d, nb in cands:
        if nb >= 0:
            i = next((i for i, e in enumerate(q) if e[1] == nb), None)
            if i is not None:
                if abs(d) < abs(q[i][2]):
                    q.pop(i)
                else:
                    continue
        q.append((z, f, d))
        q.sort()
        del q[K:]
    return q


def _oracle_list(K, cands, cid):
    """the oracle's queue fed in the clipped mesh's index order, as [(slot, sd)] (cid: slot -> clipped index)"""
    slot_of = {cid[c[0]]: c[0] for c in cands}
    fed = sorted(((float(np.float32(pz)), cid[s], float(np.float32(sd)), cid[nb] if nb >= 0 else -1) for s, pz, sd, nb in cands),
                 key=lambda t: t[1])
    return [(slot_of[f], d) for _, f, d in _oracle_queue(K, fed)]


def _clipped_view(g, F, z_clip=0.25):
    """F random faces straddling the clip plane, clipped by the oracle (pt3d.clip_faces, PyTorch3D clip.py semantics): which
    slots exist, the slot -> clipped index map, and each slot's other half.  A quad's halves are adjacent in the clipped order
    (neighbor[u2c[f]] = u2c[f] + 1), which is what frag_order_key restates."""
    fv = g.uniform(-1.0, 1.0, (F, 3, 3))
    fv[:, :, 2] = g.choice([z_clip - 0.2, z_clip + 0.3, z_clip + 0.9], (F, 3)) + g.uniform(0, 0.05, (F, 3))
    fv[F // 2, :, 2] = z_clip - 0.1                     # at least one face entirely behind the plane: culled, a gap in the order
    c = pt3d.clip_faces(torch.from_numpy(fv), torch.zeros(1, dtype=torch.long), torch.tensor([F]), z_clip, True)
    n_behind = (fv[:, :, 2] < z_clip).sum(1)
    ntri = np.array([1, 2, 1, 0])[n_behind]
    u2c, neighbor = c.u2c.numpy(), c.neighbor.numpy()
    cid, other = {}, {}
    for f in range(F):
        if ntri[f] >= 1:
            cid[f] = int(u2c[f])
            other[f] = -1
        if ntri[f] == 2:
            cid[F + f] = int(u2c[f]) + 1
            assert neighbor[cid[f]] == cid[F + f] and neighbor[cid[F + f]] == cid[f]
            other[f], other[F + f] = F + f, f
    return cid, other


@pytest.mark.parametrize('F', [7, 40, 300])
def test_order_key_is_the_clipped_index_order(fl, F):
    """frag_order_key orders the slots like the oracle's clipped face indices; frag_order_slot is its inverse"""
    g = np.random.default_rng(F)
    cid, _ = _clipped_view(g, F)
    assert any(s >= F for s in cid) and any(s not in cid for s in range(F))     # quads and culled faces both occur
    slots = sorted(cid)
    assert sorted(slots, key=lambda s: fl.hm_order_key(s, F)) == sorted(slots, key=lambda s: cid[s])
    assert [fl.hm_order_key(fl.hm_order_slot(i, F), F) for i in range(2 * F)] == list(range(2 * F))


def test_quad_halves_and_a_face_between_them_in_depth(fl):
    """K = 1; halves A = slot f and B = slot F + f of one quad, a third face C, pz_A < pz_C < pz_B and dist_B < |d_A|.
    The oracle keeps C when C's index comes after the quad (order A, B, C) and B when it comes before (C, A, B); offered in the
    list order B, C, A the list would keep A, which the oracle never keeps.  After the ordering step every list order gives
    the oracle's answer."""
    F = 10
    for c_face, want in ((7, 'C'), (1, 'B')):
        f = 4
        A, B, C = (f, 1.0, -4e-4, F + f), (F + f, 3.0, 1e-4, f), (c_face, 2.0, -5e-4, -1)
        name = {f: 'A', F + f: 'B', c_face: 'C'}
        cid = {f: 2 * f, F + f: 2 * f + 1, c_face: 2 * c_face}
        assert [name[s] for s, _ in _oracle_list(1, [A, B, C], cid)] == [want]
        assert [name[s] for s, _ in _kernel_list(fl, 1, F, RAW, [B, C, A])] == ['A']            # the order dependence
        for perm in ([A, B, C], [A, C, B], [B, A, C], [B, C, A], [C, A, B], [C, B, A]):
            for mode in (SORTED, SCANNED):
                assert [name[s] for s, _ in _kernel_list(fl, 1, F, mode, perm)] == [want], (c_face, perm, mode)


def _candidates(g, K, F, cid, other, trial):
    """one pixel's candidate set: a random subset of the view's slots (both halves of some quads, lone halves of others),
    exact depth ties on every third set, more candidates than K on most, halves inside or outside their triangle"""
    slots = np.array(sorted(cid))
    n = int(g.integers(1, min(len(slots), 3 * K + 6) + 1))
    pick = list(g.choice(slots, n, replace=False))
    # most quads that have one half here have both: the rule only acts then
    for s in list(pick):
        if other[s] >= 0 and other[s] not in pick and g.random() < 0.7:
            pick.append(other[s])
    pick = [int(s) for s in pick]
    levels = np.float32([0.5, 0.75, 1.0, 1.5])
    pz = g.uniform(0.1, 5.0, len(pick)).astype(np.float32)
    if trial % 3 == 0:
        # exact ties, broken by slot: the clipped index order, except for second halves (slot F + f) against faces g > f,
        # whose ties the list leaves in slot order (dbw_fraglist.cuh, frag_key_less): those keep distinct depths
        whole = np.array([s < F for s in pick])
        pz[whole] = g.choice(levels, int(whole.sum()))
    sd = (g.uniform(1e-6, 9e-4, len(pick)) * g.choice([-1.0, 1.0], len(pick))).astype(np.float32)
    return [(s, float(pz[i]), float(sd[i]), other[s]) for i, s in enumerate(pick)]


@pytest.mark.parametrize('K', [1, 2, 3, 10, 25])
def test_list_equals_the_oracle_queue_under_every_offer_order(fl, K):
    """random candidate sets, each offered in 60 random list orders: after the kernel's ordering step (the fast path's sort and
    the chunked path's scan order) the list equals the oracle's queue fed in the clipped mesh's index order.  Without the
    ordering step the same sets do give different lists -- the check is sensitive to what it guards."""
    g = np.random.default_rng(100 + K)
    F = 60
    cid, other = _clipped_view(g, F)
    raw_diff = checked = 0
    for trial in range(120):
        cands = _candidates(g, K, F, cid, other, trial)
        want = _oracle_list(K, cands, cid)
        for _ in range(60):
            perm = [cands[i] for i in g.permutation(len(cands))]
            for mode in (SORTED, SCANNED):
                got = _kernel_list(fl, K, F, mode, perm)
                assert got == want, (trial, mode, perm, got, want)
            raw_diff += _kernel_list(fl, K, F, RAW, perm) != want
            checked += 1
    print(f'\nK={K}: {checked} list orders, {raw_diff} of them keep other fragments when offered unsorted')
    assert raw_diff > 0
