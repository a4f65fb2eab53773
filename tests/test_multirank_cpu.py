"""CPU, world_size 2, gloo: the host-side logic of the multi-GPU force decomposition (DESIGN.md section 5).

What runs on the GPUs (kernels, NCCL) cannot run here; what CAN be checked without a GPU is the decomposition itself:
 * the term sharding rule the kernels use (work item g belongs to rank g % world) partitions every list exactly once,
 * summing the ranks' partial forces as 2^32 fixed-point int64 (the engine's all-reduce payload) reproduces the
   unsharded result bit-for-bit, independent of the rank count -- the property that lets every rank integrate the same
   trajectory,
 * the bootstrap plumbing bench.py uses (rank 0 creates a 128-byte id, broadcast to all ranks)."""
import os
import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SCALE = 4294967296.0


def _shard(desc, rank, world):
    import copy
    d = copy.copy(desc)
    sel = slice(rank, None, world)
    for names in (("exc_i", "exc_j", "exc_qq", "exc_sigma", "exc_eps"), ("bond_i", "bond_j", "bond_r0", "bond_k"),
                  ("angle_i", "angle_j", "angle_k", "angle_t0", "angle_kk")):
        for n in names:
            setattr(d, n, getattr(desc, n)[sel])
    return d


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from openmm_b200 import systems
    from oracle import port as orc
    desc = systems.water_box(4, cutoff=0.6, rigid=False).rounded()
    L = orc.lib()
    n = desc.natoms
    # bootstrap plumbing: 128-byte id from rank 0
    uid = torch.zeros(128, dtype=torch.uint8)
    if rank == 0:
        uid = torch.arange(128, dtype=torch.uint8)
    dist.broadcast(uid, 0)
    assert uid.tolist() == list(range(128))
    # sharded bonded + exception terms (rank r owns work items r, r+world, ...)
    d = _shard(desc, rank, world)
    f = np.zeros((n, 3))
    pos = orc._d(desc.positions)
    e = 0.0
    e += L.orc_bonds(len(d.bond_i), orc._ip(orc._i(d.bond_i)), orc._ip(orc._i(d.bond_j)), orc._dp(orc._d(d.bond_r0)), orc._dp(orc._d(d.bond_k)), orc._dp(pos), orc._dp(f))
    e += L.orc_angles(len(d.angle_i), orc._ip(orc._i(d.angle_i)), orc._ip(orc._i(d.angle_j)), orc._ip(orc._i(d.angle_k)), orc._dp(orc._d(d.angle_t0)),
                      orc._dp(orc._d(d.angle_kk)), orc._dp(pos), orc._dp(f))
    alpha = desc.pme_parameters()[0]
    box = orc._d(desc.box).reshape(9)
    e += L.orc_exclusion_correction(len(d.exc_i), orc._ip(orc._i(d.exc_i)), orc._ip(orc._i(d.exc_j)), orc._dp(pos), orc._dp(orc._d(desc.charges)),
                                    orc._dp(box), 0, alpha, orc._dp(f))
    fixed = torch.from_numpy(np.rint(f*SCALE).astype(np.int64))
    dist.all_reduce(fixed)                       # int64 sum: exact, order independent
    et = torch.tensor([e], dtype=torch.float64)
    dist.all_reduce(et)
    if rank == 0:
        np.save(out, np.concatenate([fixed.numpy().astype(np.float64).ravel()/SCALE, et.numpy()]))
    dist.destroy_process_group()


def test_force_decomposition_world2(tmp_path):
    from openmm_b200 import systems
    from oracle import port as orc
    out = str(tmp_path/"r.npy")
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    got = np.load(out)
    desc = systems.water_box(4, cutoff=0.6, rigid=False).rounded()
    L = orc.lib()
    n = desc.natoms
    f = np.zeros((n, 3))
    pos = orc._d(desc.positions)
    e = L.orc_bonds(len(desc.bond_i), orc._ip(orc._i(desc.bond_i)), orc._ip(orc._i(desc.bond_j)), orc._dp(orc._d(desc.bond_r0)), orc._dp(orc._d(desc.bond_k)), orc._dp(pos), orc._dp(f))
    e += L.orc_angles(len(desc.angle_i), orc._ip(orc._i(desc.angle_i)), orc._ip(orc._i(desc.angle_j)), orc._ip(orc._i(desc.angle_k)),
                      orc._dp(orc._d(desc.angle_t0)), orc._dp(orc._d(desc.angle_kk)), orc._dp(pos), orc._dp(f))
    e += L.orc_exclusion_correction(len(desc.exc_i), orc._ip(orc._i(desc.exc_i)), orc._ip(orc._i(desc.exc_j)), orc._dp(pos), orc._dp(orc._d(desc.charges)),
                                    orc._dp(orc._d(desc.box).reshape(9)), 0, desc.pme_parameters()[0], orc._dp(f))
    assert np.abs(got[:-1].reshape(n, 3) - f).max() < 3/SCALE*64        # per-term fixed-point rounding only
    assert abs(got[-1] - e) < 1e-9*abs(e)


def test_round_robin_sharding_is_a_partition():
    for world in (2, 4, 8):
        for n in (0, 1, 7, 1000, 18773):
            seen = np.zeros(n, dtype=int)
            for r in range(world):
                seen[r::world] += 1
            assert (seen == 1).all()
        # contiguous chunks for the PME atoms (k_pme_spread): per = ceil(N/world)
        N = 23558
        per = (N + world - 1)//world
        cover = np.zeros(N, dtype=int)
        for r in range(world):
            cover[r*per:min(N, (r+1)*per)] += 1
        assert (cover == 1).all()


def _role_worker(rank, world, port, out):
    """DESIGN.md section 5 at world 2: rank 0 = direct space + bonded terms + exclusion correction, rank 1 = reciprocal space
    for all atoms (what engine.cu arranges for MG_NCCL_SPLIT), joined by one int64 all-reduce of the force buffer."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from openmm_b200 import systems
    from oracle import port as orc
    desc = systems.water_box(3, cutoff=0.45, rigid=False).rounded()
    L = orc.lib()
    n = desc.natoms
    pos, q = orc._d(desc.positions), orc._d(desc.charges)
    box = orc._d(desc.box).reshape(9)
    alpha, nx, ny, nz = desc.pme_parameters()
    f = np.zeros((n, 3))
    e = 0.0
    if rank == world - 1:
        e += L.orc_pme_reciprocal(n, orc._dp(pos), orc._dp(q), orc._dp(box), alpha, nx, ny, nz, orc._dp(f))
        e += L.orc_self_energy(n, orc._dp(q), alpha)
    else:
        fd, ed, parts = orc.forces_energy(desc, pme=(alpha, nx, ny, nz))
        # everything but reciprocal space and the self term
        fr = np.zeros((n, 3))
        er = L.orc_pme_reciprocal(n, orc._dp(pos), orc._dp(q), orc._dp(box), alpha, nx, ny, nz, orc._dp(fr))
        f, e = fd - fr, ed - er - parts["self"]
    fixed = torch.from_numpy(np.rint(f*SCALE).astype(np.int64))
    dist.all_reduce(fixed)
    et = torch.tensor([e], dtype=torch.float64)
    dist.all_reduce(et)
    if rank == 0:
        np.save(out, np.concatenate([fixed.numpy().astype(np.float64).ravel()/SCALE, et.numpy()]))
    dist.destroy_process_group()


def test_role_split_direct_rank_plus_reciprocal_rank_world2(tmp_path):
    from openmm_b200 import systems
    from oracle import port as orc
    out = str(tmp_path/"role.npy")
    port = 31500 + (os.getpid() % 2000)
    mp.spawn(_role_worker, args=(2, port, out), nprocs=2, join=True)
    got = np.load(out)
    desc = systems.water_box(3, cutoff=0.45, rigid=False).rounded()
    f, e, _ = orc.forces_energy(desc)
    assert np.abs(got[:-1].reshape(desc.natoms, 3) - f).max() < 1e-6      # int64 rounding of two partial sums + one subtraction
    assert abs(got[-1] - e) < 1e-9*abs(e)


# ---- the round-2 scheme: owner decomposition over a peer-memory data plane (DESIGN.md section 5) ----
def owner_cuts(unit_atoms, natoms, world):
    """engine.cu:setup_ownership restated: cut the atom range at integration-unit boundaries, balanced by atom count; a cut
    is only legal where the units before it hold exactly the atoms below some index."""
    U = len(unit_atoms)
    lo = np.array([min(a for a in u if a >= 0) for u in unit_atoms]); hi = np.array([max(u) for u in unit_atoms])
    pref_max = np.concatenate([[-1], np.maximum.accumulate(hi)])
    suf_min = np.concatenate([np.minimum.accumulate(lo[::-1])[::-1], [natoms]])
    atom_lo, unit_lo, u = [0], [0], 1
    for q in range(1, world):
        target = q*natoms//world
        while u < U and not (pref_max[u] < suf_min[u] and suf_min[u] >= target):
            u += 1
        assert u < U
        unit_lo.append(u); atom_lo.append(int(suf_min[u])); u += 1
    return atom_lo + [natoms], unit_lo + [U]


def test_owner_cuts_respect_integration_units():
    # 40 waters (O, H, H) after a 7-atom "solute" of single-atom units and one X-H3 cluster
    units = [(0,), (1,), (2, 3, 4, 5), (6,)] + [(7 + 3*w, 8 + 3*w, 9 + 3*w) for w in range(40)]
    n = 7 + 120
    for world in (2, 3, 4, 8):
        atom_lo, unit_lo = owner_cuts(units, n, world)
        assert atom_lo[0] == 0 and atom_lo[-1] == n and all(b > a for a, b in zip(atom_lo, atom_lo[1:]))
        for q in range(world):
            owned = set(a for u in units[unit_lo[q]:unit_lo[q+1]] for a in u)
            assert owned == set(range(atom_lo[q], atom_lo[q+1]))          # whole units, contiguous atoms
        sizes = np.diff(atom_lo)
        assert sizes.max() - sizes.min() <= 6                              # balanced to within two units


def _owner_worker(rank, world, port, out):
    """One evaluation + one 'integrate' of the owner scheme with gloo standing in for the NVLink stores: every rank computes
    PARTIAL fixed-point forces on all atoms (its share of the work items), sends each owner the partials of the owner's atoms
    (k_force_push -> inbox), the owner totals them exactly (k_integrate), moves ITS atoms and hands the new positions to
    everybody (the position stores of k_integrate); the charge grid is reduced slab by slab to the slab owners (k_grid_push +
    the summation in k_fft_slab_fwd)."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(11)
    n, nwork, nx = 96, 1000, 12
    units = [(3*w, 3*w + 1, 3*w + 2) for w in range(n//3)]
    atom_lo, unit_lo = owner_cuts(units, n, world)
    pos = rng.standard_normal((n, 3))
    wi, wj = rng.integers(0, n, nwork), rng.integers(0, n, nwork)
    wf = rng.standard_normal((nwork, 3))*100
    # partial forces of this rank's work items (item g -> rank g % world), 2^32 fixed point like the device buffer
    part = np.zeros((n, 3), dtype=np.int64)
    for g in range(rank, nwork, world):
        fx = np.rint(wf[g]*SCALE).astype(np.int64)
        part[wi[g]] += fx; part[wj[g]] -= fx
    # inbox exchange: all_to_all of the owner ranges
    send = [torch.from_numpy(part[atom_lo[q]:atom_lo[q+1]].copy()) for q in range(world)]
    recv = [torch.zeros((atom_lo[rank+1] - atom_lo[rank], 3), dtype=torch.int64) for _ in range(world)]
    for q in range(world):                      # gloo has no all_to_all on CPU tensors of unequal size everywhere: point to point
        if q == rank:
            recv[q] = send[q]
        elif rank < q:
            dist.send(send[q], q); dist.recv(recv[q], q)
        else:
            dist.recv(recv[q], q); dist.send(send[q], q)
    total_own = sum(r.numpy() for r in recv)                          # exact integer sum, any order
    # owner integrates its atoms and publishes them
    newpos = pos.copy()
    newpos[atom_lo[rank]:atom_lo[rank+1]] += 1e-3*total_own.astype(np.float64)/SCALE
    gathered = [torch.zeros((atom_lo[q+1] - atom_lo[q], 3), dtype=torch.float64) for q in range(world)]
    for q in range(world):
        t = torch.from_numpy(newpos[atom_lo[q]:atom_lo[q+1]].copy()) if q == rank else gathered[q]
        dist.broadcast(t, q)
        gathered[q] = t
    allpos = np.concatenate([g.numpy() for g in gathered])
    # charge grid: every rank spreads ITS atoms into a full grid, slabs go to their owners and are summed there
    grid = np.zeros((nx, 4, 4), dtype=np.int64)
    for a in range(atom_lo[rank], atom_lo[rank+1]):
        grid[int(abs(pos[a, 0])*3) % nx, a % 4, (a//4) % 4] += np.int64(round(pos[a, 1]*SCALE))
    x_lo = [q*nx//world for q in range(world + 1)]
    slab = torch.from_numpy(grid.copy())
    dist.all_reduce(slab)                                             # what the slab owners end up with, restricted to their planes
    mine = slab.numpy()[x_lo[rank]:x_lo[rank+1]]
    if rank == 0:
        np.savez(out, pos=allpos, plane_sum=int(mine.sum()), atom_lo=np.array(atom_lo))
    dist.destroy_process_group()


def test_owner_decomposition_protocol_world2(tmp_path):
    out = str(tmp_path/"owner.npz")
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_owner_worker, args=(2, port, out), nprocs=2, join=True)
    z = np.load(out)
    # the single-rank answer
    rng = np.random.default_rng(11)
    n, nwork = 96, 1000
    pos = rng.standard_normal((n, 3))
    wi, wj = rng.integers(0, n, nwork), rng.integers(0, n, nwork)
    wf = rng.standard_normal((nwork, 3))*100
    tot = np.zeros((n, 3), dtype=np.int64)
    for g in range(nwork):
        fx = np.rint(wf[g]*SCALE).astype(np.int64)
        tot[wi[g]] += fx; tot[wj[g]] -= fx
    expect = pos + 1e-3*tot.astype(np.float64)/SCALE
    assert np.array_equal(z["pos"], expect)                           # bit-identical to one rank: integer sums commute


def test_engine_ownership_cuts_on_the_real_systems_match_the_model():
    """b200md_ownership_probe runs the engine's own classification + cuts (no device): on DHFR and ApoA1 every rank owns whole
    integration units, the ranges partition the atoms, they are balanced to a few atoms, and they equal owner_cuts() above."""
    import ctypes as C
    from conftest import ROOT
    from openmm_b200 import systems, _lib
    lib = _lib.load()
    D, I = C.POINTER(C.c_double), C.POINTER(C.c_int)
    for name in ("dhfr", "apoa1"):
        d = systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz"))
        n = d.natoms
        mass = np.ascontiguousarray(d.masses, np.float64)
        ci, cj, cd = np.ascontiguousarray(d.con_i, np.int32), np.ascontiguousarray(d.con_j, np.int32), np.ascontiguousarray(d.con_d, np.float64)
        # the model's units: SETTLE waters / X-H_n clusters / single atoms, from the constraint graph
        adj = [[] for _ in range(n)]
        for a, b in zip(ci, cj):
            adj[a].append(int(b)); adj[b].append(int(a))
        seen, units = np.zeros(n, bool), []
        for a in range(n):
            if seen[a]:
                continue
            comp, stack = [], [a]
            seen[a] = True
            while stack:
                x = stack.pop(); comp.append(x)
                for y in adj[x]:
                    if not seen[y]:
                        seen[y] = True; stack.append(y)
            units.append(tuple(sorted(comp)))
        units.sort()
        for world in (2, 4, 8):
            alo = np.zeros(world + 1, np.int32); ulo = np.zeros(world + 1, np.int32)
            nu = lib.b200md_ownership_probe(n, mass.ctypes.data_as(D), len(ci), ci.ctypes.data_as(I), cj.ctypes.data_as(I), cd.ctypes.data_as(D),
                                            world, alo.ctypes.data_as(I), ulo.ctypes.data_as(I))
            assert nu == len(units)
            m_alo, m_ulo = owner_cuts(units, n, world)
            assert list(alo) == m_alo and list(ulo) == m_ulo
            sizes = np.diff(alo)
            assert sizes.min() > 0 and sizes.max() - sizes.min() <= 8


def test_octet_rotation_schedule_of_the_tile_kernel_visits_every_pair_once():
    """Index logic of nonbonded.cu:pair_tiles restated: four groups of eight rotations inside 8-lane octets, then the octets move
    on by 8 lanes.  Every (i lane, j slot) pair must be met exactly once, the mask bit consumed must be that slot's, and after the
    last rotation every j (and its force total) must be back in its home lane."""
    holder = list(range(32))                    # holder[lane] = home lane (slot) of the j atom the lane holds
    met = np.zeros((32, 32), int)
    for g in range(4):
        slot_base = [(((lane >> 3) + g) & 3) << 3 for lane in range(32)]
        for k in range(8):
            for lane in range(32):
                slot = slot_base[lane] | (((lane & 7) + k) & 7)         # what the kernel uses for the mask bit and the close-pair queue
                assert holder[lane] == slot
                met[lane, slot] += 1
            holder = [holder[(lane & ~7) | ((lane + 1) & 7)] for lane in range(32)]      # srcIn
        assert all(holder[lane] == slot_base[lane] | (lane & 7) for lane in range(32))    # the octet is home again: sums are folded
        holder = [holder[(lane + 8) & 31] for lane in range(32)]                          # srcOut
    assert (met == 1).all()
    assert holder == list(range(32))
