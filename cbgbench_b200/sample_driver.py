"""Sampling driver: the CUDA (H100) counterpart of the reference's ``sample.py`` loop (SURVEY.md section 8 row f1).

Mirrors the reference's sample.py:159-241 for the part that belongs to the hot path: build mini-batches
of pocket+ligand graphs, ``model.sample(batch)``, take ``traj[0]`` (the state the reference consumes,
sample.py:194-201), split it per pocket (``split_batch_into_samples``, sample.py:16-32) and collect
``{pos, v}`` per ligand.  What stays outside: LMDB/PDB parsing and RDKit/OpenBabel reconstruction (CPU
chemistry tooling, out of scope, DESIGN.md section 9) - pockets are synthetic (``cbgbench_b200.synthetic``)
or come from a ``torch.save``d list of batch dicts with the reference's keys.

Multi-GPU (torchrun, one rank per GPU): every mini-batch's pockets are partitioned over the ranks by atom
count, each rank samples its share with no communication and ONE all-gather returns the final
coordinates / types (``cbgbench_b200.sharding``).

    python -m cbgbench_b200.sample_driver --pockets 16 --batch-size 16 --out out.pt
    python -m cbgbench_b200.sample_driver --builder device --size-prior <reference>/repo/datasets/transforms/_atom_num_dist.npy \
        --pockets 2 --num-samples 100 --batch-size 50      (row f3: batches built on the GPU from raw pockets,
                                                            sample.py:177-183: num_samples per pocket, batch_size per step)
    python -m cbgbench_b200.sample_driver --model diffsbdd --pockets 16      (row f2: also diffbp)
    python -m cbgbench_b200.sample_driver --model difffg --pockets 16 --n-prot 100 --n-lig 12
                                        (D3FG: --n-prot residues and --n-lig functional groups per pocket, one GPU)
    torchrun --nproc-per-node 8 -m cbgbench_b200.sample_driver --pockets 512 --batch-size 512
"""
import argparse
import os
import time

import torch

from . import sharding, synthetic
from .targetdiff import TargetDiffB200
from .diffsbdd import DiffSBDDB200
from .diffbp import DiffBPB200
from .difffg import D3FGB200

MODELS = {'targetdiff': (TargetDiffB200, synthetic.targetdiff_config),
          'diffsbdd': (DiffSBDDB200, synthetic.diffsbdd_config),
          'diffbp': (DiffBPB200, synthetic.diffbp_config),
          'difffg': (D3FGB200, synthetic.difffg_config)}


def split_batch_into_samples(x, v, graph_id, n_graphs):
    """Per-pocket results of one mini-batch (sample.py:16-32): list of dicts {pos [n,3], v [n]}."""
    out = []
    for g in range(n_graphs):
        m = graph_id == g
        out.append({'pos': x[m].cpu(), 'v': v[m].cpu()})
    return out


def split_batch_into_samples_fg(xc, c, o, graph_id, n_graphs):
    """Per-pocket D3FG results (sample.py:34-47, no translation: d3fg_fg.yml sets translate false): list of dicts
    {pos_center [n,3], fg_type [n], orientation [n,3]}."""
    out = []
    for g in range(n_graphs):
        m = graph_id == g
        out.append({'pos_center': xc[m].cpu(), 'fg_type': c[m].argmax(-1).cpu(), 'orientation': o[m].cpu()})
    return out


def run_difffg(args, model, distributed):
    if distributed:
        raise SystemExit('sample_driver --model difffg runs on one GPU: D3FG pockets are not sharded over ranks')
    results, t0 = [], time.time()
    for b0 in range(0, args.pockets, args.batch_size):
        nb = min(args.batch_size, args.pockets - b0)
        batch = synthetic.make_fg_batch([args.n_prot] * nb, [args.n_lig] * nb, seed=args.seed + b0)
        xc, c, o, gid = model.sample(batch, traj_mode='final')[0]
        results.extend(split_batch_into_samples_fg(xc, c, o, gid, nb))
    torch.cuda.synchronize()
    dt = time.time() - t0
    if args.out:
        torch.save(results, args.out)
    print(f'sampled {len(results)} FG sets in {dt:.2f} s ({len(results) / dt:.2f} pockets/s, {args.steps} steps)')
    return results


def final_state(model, sub_batch, traj_key=0):
    """model.sample on a (sub-)batch -> (x, v) of traj[traj_key] on the model's device."""
    traj = model.sample(sub_batch, traj_mode='final')
    x, c, _ = traj[traj_key]
    dev = next(model.parameters()).device
    return x.to(dev), c.argmax(-1).to(dev)


def device_built_batches(args, dev):
    """Row f3: the transform list of configs/denovo/test/<model>.yml evaluated on the GPU (DeviceBatchBuilder) for
    synthetic RAW pockets: every pocket is sampled --num-samples times in mini-batches of --batch-size samples, like
    sample.py:177-183 (``data_list_repeat`` + DataLoader).  Generator: torch's CUDA generator (seeded by --seed)."""
    import numpy as np
    from .batch_builder import DeviceBatchBuilder, SizePrior
    if not args.size_prior:
        raise SystemExit('--builder device needs --size-prior (the reference\'s _atom_num_dist.npy)')
    prior = SizePrior.from_npy(args.size_prior)
    recipe = {'targetdiff': dict(type_dist='uniform', pos_dist='gaussian', num_classes=13),
              'diffbp': dict(type_dist='absorbing', pos_dist='gaussian', num_classes=13),
              'diffsbdd': dict(type_dist='zeros', pos_dist='zero_mean_gaussian', num_classes=13)}[args.model]
    builder = DeviceBatchBuilder(prior, recipe='denovo', **recipe)
    rs = np.random.RandomState(args.seed)
    batches = []
    for _ in range(args.pockets):
        n = args.n_prot
        pocket = {'pos': torch.from_numpy((rs.normal(0, 5.0, size=(n, 3)) + rs.normal(0, 20, size=3)).astype(np.float32)),
                  'element': torch.from_numpy(rs.choice([1, 6, 7, 8, 16], size=n, p=[0.05, 0.55, 0.18, 0.2, 0.02])),
                  'is_backbone': torch.from_numpy(rs.randint(0, 2, size=n).astype(bool)),
                  'atom_to_aa_type': torch.from_numpy(rs.randint(0, 20, size=n))}
        for s0 in range(0, args.num_samples, args.batch_size):
            b = builder.build([pocket], min(args.batch_size, args.num_samples - s0), device=dev)
            if args.model == 'diffsbdd':          # our DiffSBDD host class takes integer types like the other two
                b['ligand_atom_type'] = torch.zeros(b['ligand_pos'].shape[0], dtype=torch.int64, device=dev)
            batches.append(b)
    return batches


def run(args):
    distributed = int(os.environ.get('WORLD_SIZE', '1')) > 1
    rank = int(os.environ.get('RANK', '0'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    dev = torch.device('cuda', local_rank)
    torch.cuda.set_device(dev)
    if distributed and not torch.distributed.is_initialized():
        torch.distributed.init_process_group('nccl', device_id=dev)
    cls, make_cfg = MODELS[args.model]                                                     # get_model(cfg), sample.py:155
    model = cls(make_cfg(num_steps=args.steps, num_layers=args.layers))
    if args.ckpt:
        ckpt = torch.load(args.ckpt, map_location='cpu')
        model.load_state_dict(ckpt['model'] if 'model' in ckpt else ckpt, strict=True)     # sample.py:153-157
    else:
        model.load_state_dict(synthetic.seeded_state_dict(model, seed=0), strict=True)
    model = model.to(dev).eval()
    torch.manual_seed(args.seed + rank)                                                    # sample.py:106,131-133
    if args.model == 'difffg':
        return run_difffg(args, model, distributed)

    if args.builder == 'device':
        batches = device_built_batches(args, dev)
    elif args.batches:
        batches = torch.load(args.batches)
    else:
        batches = []
        for b0 in range(0, args.pockets, args.batch_size):
            nb = min(args.batch_size, args.pockets - b0)
            b = synthetic.make_batch([args.n_prot] * nb, [args.n_lig] * nb, seed=args.seed + b0, gen_mode=args.gen_mode)
            if args.model == 'diffbp':        # configs/denovo/test/diffbp.yml:19-21 assign_atomtype: absorbing
                b['ligand_atom_type'] = torch.zeros_like(b['ligand_atom_type'])
            batches.append(b)
    results, t0 = [], time.time()
    for batch in batches:
        n_graphs = int(batch['ligand_element_batch'].max()) + 1
        if distributed:
            x, v, gid = sharding.sample_sharded(lambda sub: final_state(model, sub), batch)
        else:
            x, v = final_state(model, batch)
            gid = batch['ligand_element_batch'].to(x.device)
        # translate back like sample.py:198-201, per graph (the reference adds protein_translation[:1] to the whole batch,
        # identical for its batches of copies of one pocket; synthetic pockets are already centred: no translation)
        tr = sharding.graph_translation(batch)
        if tr is not None:
            x = x + tr.to(x.device)[gid]
        results.extend(split_batch_into_samples(x, v, gid, n_graphs))
    torch.cuda.synchronize()
    dt = time.time() - t0
    if rank == 0:
        if args.out:
            torch.save(results, args.out)
        print(f'sampled {len(results)} ligands in {dt:.2f} s ({len(results) / dt:.2f} ligands/s, '
              f'{args.steps} steps, world {int(os.environ.get("WORLD_SIZE", "1"))})')
    if distributed:
        torch.distributed.barrier()
    return results


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--model', default='targetdiff', choices=sorted(MODELS))
    ap.add_argument('--pockets', type=int, default=16)
    ap.add_argument('--batch-size', type=int, default=16)          # sample.py:108
    ap.add_argument('--n-prot', type=int, default=300)
    ap.add_argument('--n-lig', type=int, default=24)
    ap.add_argument('--gen-mode', default='denovo', choices=['denovo', 'partial'])
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--layers', type=int, default=9)
    ap.add_argument('--seed', type=int, default=2024)               # sample.py:106
    ap.add_argument('--ckpt', default=None, help='reference checkpoint ({"model": state_dict, ...})')
    ap.add_argument('--batches', default=None, help='torch.save()d list of batch dicts with the reference keys')
    ap.add_argument('--out', default=None)
    ap.add_argument('--builder', default='host', choices=['host', 'device'],
                    help="'device': build the batches on the GPU from raw pockets (row f3)")
    ap.add_argument('--size-prior', default=None, help='path of the reference size-prior table (_atom_num_dist.npy)')
    ap.add_argument('--num-samples', type=int, default=8, help='samples per pocket with --builder device (sampling.num_samples)')
    return run(ap.parse_args(argv))


if __name__ == '__main__':
    main()
