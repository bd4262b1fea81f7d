"""Experiment driver: same command line, artefacts and metrics line as the reference's main.py
(reference main.py:8-41 flags, :44-187 main), running on the native engine.

Flags added here (all excluded from the result-directory name so layouts stay compatible):
--synthetic N, --random_init, --max_iterations, --sampling_size, --num_batches, --precision,
--chunk, --img_size, --seed, --pc_n_patch, --attack_pc_n_patch, --basic_unit, --eot_sampler, --checkpoint_every.

--pc_n_patch 2 evaluates against the two-patch PatchCleanser (MaskWindow(img, r, 2), reference
defenses/PatchCleanser.py:34-37).  It does not change the generated patches, so a run on an existing
result directory reuses them; its records go to adv_PC2_<i>.pt, apart from the one-patch adv_PC_<i>.pt.

--attack_pc_n_patch 2 generates the patches against that window (DorPatch.generate(pc_n_patch=2)).  It changes the
artefacts, so it is the exception to the rule above: the first path component gets `__attack_pc_n_patch=2`, and a
two-patch run never resumes from, or overwrites, one-patch patches.  The usual run sets both flags to 2.

--basic_unit N (default 7, the reference's) sets the side of the square cells the group lasso and patch_selection work
on (DorPatch.generate(basic_unit=N)); it must divide the image size.  It changes the patches and the stage-0 mask, so a
non-default unit is also appended to the first path component (`__basic_unit=N`).

--eot_sampler device draws generate()'s EOT occlusions on the GPU (DorPatch.generate(eot_sampler="device")): seeded and
reproducible, but not numpy's stream, so the patches differ from a host-sampler run.  It is appended to the first path
component (`__eot_sampler=device`), so such a run has its own results and stage-0 cache.

--checkpoint_every N (default 0: off) makes every batch's generate() resumable: batch i keeps its state in
<result_dir>/adv_ckpt_<i>.pt every N steps (DorPatch.generate(checkpoint=..., checkpoint_every=N)).  A rerun with the same
flags skips the finished batches, continues the interrupted one from its checkpoint and, since the checkpoint restores the
RNG streams, computes what the uninterrupted run would have.  It changes nothing that is computed, so it stays out of the
result path.

Under torchrun the PatchCleanser evaluation is sharded too (PatchCleanser(..., shard=True)): each rank forwards a share of
every robust_predict call and the labels are gathered, so every rank holds the single-process records and rank 0 writes them (DESIGN section 5).
"""
import argparse
import os
import pickle

import numpy as np
import torch
from tqdm import tqdm

from .attack import DorPatch
from .defenses.PatchCleanser import MaskWindow, PatchCleanser
from .utils import (NUM_CLASSES_DICT, NormModel, convert_float_list_to_str, generate_saving_path, get_dataset,
                    get_model, get_normalize, set_device, set_random_seed, unwrap_native)

parser = argparse.ArgumentParser(description='set parameters for patch generation')
parser.add_argument('--device', default='0', type=str, metavar='DEVICE', help='gpu device id')
parser.add_argument('--dataset', '-d', default='imagenet', type=str, metavar='DATASET', help='dataset',
                    choices=['cifar10', 'imagenet', 'cifar100'])
parser.add_argument('--data_dir', default='/home/data/data', help='path to dataset')
parser.add_argument('--model_dir', default='pretrained_models/', help='path to model')
parser.add_argument('--base_arch', '-ba', metavar='BARCH', default='resnetv2', choices=['resnetv2'],
                    help='base model architecture for patch generation (default: resnetv2)')
parser.add_argument('--targeted', '-t', action='store_true', help='targeted attack or not')
parser.add_argument('--patch_budget', default=0.12, type=float, help='patch budget')
parser.add_argument('--attack', '-a', default='DorPatch', type=str, metavar='ATTACK', help='atttack method',
                    choices=['DorPatch'])
parser.add_argument('-b', '--batch-size', default=1, type=int, metavar='N', help='mini-batch size (default: 64)')
parser.add_argument('-e', '--epsilon', default=4., type=float, metavar='E',
                    help='epsilon to bound the perturbation (l2 norm)')
parser.add_argument('--lr', '--learning-rate', default=0.01, type=float, metavar='LR', help='initial learning rate')
# settings for DorPatch
parser.add_argument('--num_patch', default=-1, type=int, help='number of patches (default: -1 as unconstrained)')
parser.add_argument('--dropout', default=2, type=int,
                    help='using how many rounds of image dropout (for robustness to occlusion)')
parser.add_argument('--density', default=1e-3, type=float,
                    help='the coeff of density regularization (for distributed property) or not')
parser.add_argument('--structured', default=1e-3, type=float, help='the coeff of structured loss')
# ---- additions (not part of the result path) ----
parser.add_argument('--synthetic', default=0, type=int, help='use N synthetic images instead of a dataset')
parser.add_argument('--random_init', action='store_true', help='random-init classifier (no checkpoint)')
parser.add_argument('--max_iterations', default=5000, type=int, help='iterations per stage (reference: 5000)')
parser.add_argument('--sampling_size', default=128, type=int, help='EOT occlusion samples per step (reference: 128)')
parser.add_argument('--num_batches', default=10, type=int, help='number of batches to attack (reference: 10)')
parser.add_argument('--precision', default=None, choices=['fp32', 'tf32', 'bf16'], help='engine arithmetic')
parser.add_argument('--chunk', default=None, type=int, help='samples per classifier pass')
parser.add_argument('--img_size', default=224, type=int, help='synthetic image size (multiple of 56)')
parser.add_argument('--seed', default=0, type=int, help='seed of the random-init weights')
parser.add_argument('--pc_n_patch', default=1, type=int, choices=[1, 2],
                    help='patches the PatchCleanser evaluation is provisioned for (2: records in adv_PC2_<i>.pt)')
parser.add_argument('--attack_pc_n_patch', default=1, type=int, choices=[1, 2],
                    help='patches of the PatchCleanser window the EOT occlusions are drawn from (2: result path suffix)')
parser.add_argument('--basic_unit', default=7, type=int,
                    help='side of the group-lasso / patch-selection cells, dividing the image size (non-7: path suffix)')
parser.add_argument('--eot_sampler', default='host', choices=['host', 'device'],
                    help="where generate() draws the EOT occlusions: 'host' (numpy, the reference's stream) or 'device' "
                         "(seeded counter-based draws on the GPU; non-host: path suffix)")
parser.add_argument('--checkpoint_every', default=0, type=int,
                    help='resumable generation: save each batch\'s attack state to <result_dir>/adv_ckpt_<i>.pt every N '
                         'steps (0: off)')


def _init_distributed():
    """Under torchrun (RANK / WORLD_SIZE / LOCAL_RANK set): one process per GPU, NCCL process group, the EOT axis of
    every generate() call and the masked forwards of every robust_predict call sharded over the ranks (attack._dist).
    Returns (rank, world)."""
    if "RANK" not in os.environ or int(os.environ.get("WORLD_SIZE", "1")) < 2:
        return 0, 1
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return dist.get_rank(), dist.get_world_size()


def main(args):
    rank, world = 0, 1
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        rank, world = _init_distributed()        # the launcher assigned the GPU: --device is not applied
    else:
        set_device(args.device)
    set_random_seed()
    if args.precision:
        os.environ["DORPATCH_PRECISION"] = args.precision
    if args.chunk:
        os.environ["DORPATCH_CHUNK"] = str(args.chunk)
    result_dir = generate_saving_path(vars(args).copy())
    if world > 1:
        import torch.distributed as dist

    def sync_ranks():
        if world > 1:
            dist.barrier()

    model = get_model(args.dataset, args.base_arch, args.model_dir, random_init=args.random_init, seed=args.seed)
    model = NormModel(model, get_normalize(args.dataset, args.base_arch))
    model = torch.nn.DataParallel(model)      # kept for interface parity; the native path unwraps it
    model.cuda()
    model.eval()
    net = unwrap_native(model)

    dataloader = get_dataset(args.dataset, data_dir=args.data_dir, batch_size=args.batch_size,
                             synthetic=args.synthetic, img_size=args.img_size)
    attack = DorPatch()
    img = args.img_size if args.synthetic else 224
    # shard=True: every rank evaluates every image below, so robust_predict shares the forwards over the ranks
    defense = [PatchCleanser(MaskWindow(img, r, args.pc_n_patch), model, shard=True) for r in [0.015, 0.03, 0.06, 0.12]]
    pc_name = "adv_PC_%d.pt" if args.pc_n_patch == 1 else "adv_PC2_%d.pt"

    target_list, preds_list, y_list, preds_adv_list, records = [], [], [], [], []
    with torch.no_grad():
        for i, (x, y) in tqdm(enumerate(dataloader)):
            if i == args.num_batches:
                break
            x = x.cuda()
            y = y.cuda()
            eng = net.engine(x.shape[-1], max_images=x.shape[0])
            preds = torch.from_numpy(eng.predict(x.contiguous().float()).astype(np.int64)).cuda()
            if args.synthetic:
                y = preds.clone()             # synthetic labels: the clean prediction is "correct" by definition
            correct = (preds == y)
            if correct.sum() == 0:
                continue
            x, y, preds = x[correct].contiguous(), y[correct], preds[correct]

            if os.path.exists(os.path.join(result_dir, "adv_mask_%d.pt" % i)):
                adv_mask = torch.load(os.path.join(result_dir, "adv_mask_%d.pt" % i)).cuda()
                adv_pattern = torch.load(os.path.join(result_dir, "adv_pattern_%d.pt" % i)).cuda()
                if args.targeted:   # recover the target label from stage 0 (main.py:108-118)
                    dir_0 = os.path.dirname(result_dir.rstrip('/'))
                    m0 = torch.load(os.path.join(dir_0, "adv_mask_%d.pt" % i)).cuda()
                    p0 = torch.load(os.path.join(dir_0, "adv_pattern_%d.pt" % i)).cuda()
                    adv_x_0, _, _ = eng.paste(x, m0, p0, args.epsilon)
                    target_list.append(eng.predict(adv_x_0).astype(np.int64))
                    assert (target_list[-1] != y.cpu().numpy()).all()
            else:
                target = None
                if args.targeted:
                    target = torch.randint(0, NUM_CLASSES_DICT[args.dataset], x.shape[:1]).cuda()
                    assert (target != y).all()
                    target_list.append(target.cpu().numpy())
                adv_mask, adv_pattern = attack.generate(
                    model, x, args.patch_budget, NUM_CLASSES_DICT[args.dataset], targeted=args.targeted,
                    y=target if args.targeted else None, lr=args.lr, num_patch=args.num_patch, dropout=args.dropout,
                    density=args.density, structured=args.structured, save_dir=result_dir, batch_id=i,
                    eps=args.epsilon, max_iterations=args.max_iterations, sampling_size=args.sampling_size,
                    pc_n_patch=args.attack_pc_n_patch, basic_unit=args.basic_unit, eot_sampler=args.eot_sampler,
                    checkpoint=os.path.join(result_dir, "adv_ckpt_%d.pt" % i) if args.checkpoint_every > 0 else None,
                    checkpoint_every=args.checkpoint_every)
                if rank == 0:                     # every rank holds the identical result; one writer
                    torch.save(adv_mask, os.path.join(result_dir, "adv_mask_%d.pt" % i))
                    torch.save(adv_pattern, os.path.join(result_dir, "adv_pattern_%d.pt" % i))
                sync_ranks()

            adv_x, _, _ = eng.paste(x, adv_mask, adv_pattern, args.epsilon)

            pc_path = os.path.join(result_dir, pc_name % i)
            if os.path.exists(pc_path):
                with open(pc_path, 'rb') as f:
                    records_batch = pickle.load(f)
            else:
                records_batch = [[d.robust_predict(im, True) for d in defense] for im in adv_x]
                if rank == 0:
                    with open(pc_path, 'wb') as f:
                        pickle.dump(records_batch, f)
                sync_ranks()

            preds_list.append(preds.cpu().numpy())
            y_list.append(y.cpu().numpy())
            preds_adv_list.append(eng.predict(adv_x).astype(np.int64))
            records += records_batch

    if args.targeted:
        target_list = np.concatenate(target_list)
    preds_list = np.concatenate(preds_list)
    y_list = np.concatenate(y_list)
    preds_adv_list = np.concatenate(preds_adv_list)
    acc_clean = (preds_list == y_list).mean() * 100
    acc_robust = (preds_adv_list == y_list).mean() * 100
    for k, d in enumerate(defense):
        d.collect([r[k] for r in records])
    pred_prov = [d.result.predictions for d in defense]
    certifiable = [d.result.certifications for d in defense]
    acc_PC = [(p == y_list).mean() * 100 for p in pred_prov]
    certified_acc_PC = [((p == y_list) & c).mean() * 100 for p, c in zip(pred_prov, certifiable)]
    if args.targeted:
        certified_asr_PC = [((p == target_list) & c).mean() * 100 for p, c in zip(pred_prov, certifiable)]
    else:
        certified_asr_PC = [((p != y_list) & c).mean() * 100 for p, c in zip(pred_prov, certifiable)]
    line = "clean accuracy: {:.2f}%, robust accuracy:{:.2f}%, acc@PC:{:s}%, certified_ACC@PC:{:s}%, certified_ASR@PC:{:s}%".format(
        acc_clean, acc_robust, convert_float_list_to_str(acc_PC), convert_float_list_to_str(certified_acc_PC),
        convert_float_list_to_str(certified_asr_PC))
    if rank == 0:
        print(line)
    return dict(acc_clean=acc_clean, acc_robust=acc_robust, acc_PC=acc_PC, certified_acc_PC=certified_acc_PC,
                certified_asr_PC=certified_asr_PC, result_dir=result_dir, line=line)


def cli(argv=None):
    return main(parser.parse_args(argv))


if __name__ == '__main__':
    cli()
