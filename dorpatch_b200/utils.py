"""Host-side mirror of the reference's utils.py (same names, arguments and error behaviour).

Reference: reference utils.py -- set_device :12-13, set_random_seed :16-21,
generate_saving_path :24-44, get_model :47-63, get_normalize :66-68, NormModel :71-78,
get_dataset :81-102, clip :105-110, convert_float_list_to_str :112.
Compute (`clip`, the classifier) runs in libdorpatch.so; this file is glue.
"""
import json
import os
import random

import numpy as np
import torch

from .resnetv2 import ResNetV2

NUM_CLASSES_DICT = {'imagenet': 1000, 'cifar10': 10, 'cifar100': 100}


def set_device(device):
    os.environ['CUDA_VISIBLE_DEVICES'] = device


def set_random_seed(seed=1234):
    random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)
    np.random.seed(seed)


# flags added by this implementation; excluded from the result path so that directory
# layouts (and therefore resume) stay compatible with the reference's
EXTRA_FLAGS = ("synthetic", "random_init", "max_iterations", "sampling_size", "num_batches",
               "precision", "chunk", "img_size", "seed", "pc_n_patch", "attack_pc_n_patch", "basic_unit")


# extra flags that change WHAT is computed (and therefore the artefacts a later run would resume from), with the
# value at which the run is the reference's: any other value is appended to the first path component, so a
# synthetic / random-init / truncated run can never be resumed as (or shadow) a real one.  precision / chunk /
# num_batches do not change the artefacts' meaning and stay out of the path.
ARTEFACT_FLAGS = (("synthetic", 0), ("random_init", False), ("max_iterations", 5000), ("sampling_size", 128),
                  ("img_size", 224), ("seed", 0), ("attack_pc_n_patch", 1), ("basic_unit", 7))


def generate_saving_path(configs):
    """results/<k=v joined by _>/num_patch=.._patch_budget=..  (utils.py:24-44).  With the reference's flag values the
    path is the reference's; non-default values of the flags in ARTEFACT_FLAGS add a `__k=v_...` suffix."""
    json.dumps(configs, indent=4)
    extra = ["%s=%s" % (k, configs[k]) for k, d in ARTEFACT_FLAGS if k in configs and configs[k] != d]
    for k in ["device", "model_dir", "data_dir", "batch_size", "lr", "epsilon"] + list(EXTRA_FLAGS):
        configs.pop(k, None)
    subdir = ''
    if configs["attack"] == 'DorPatch':
        parts = []
        for k in ["num_patch", "patch_budget"]:
            parts.append("%s=%s" % (k, configs.pop(k)))
        subdir = '_'.join(parts)
    print(subdir)
    top = "_".join("%s=%s" % (k, v) for k, v in configs.items())
    if extra:
        top += "__" + "_".join(extra)
    save_path = os.path.join("results", top, subdir)
    os.makedirs(save_path, exist_ok=True)
    return save_path


def get_model(dataset_name, model_name, model_dir='pretrained_models', random_init=False, seed=0):
    """utils.py:47-63.  `resnetv2` resolves to the in-repo ResNetV2-50x1-BiT container (timm
    is not a dependency).  With random_init=False the PatchCleanser checkpoint
    ``<model_dir>/<dataset>/resnetv2_50x1_bit_distilled_cutout2_128_<dataset>.pth`` is loaded
    exactly as the reference does; a missing file raises (FileNotFoundError), as there."""
    names = ['resnetv2_50x1_bit_distilled', 'vit_base_patch16_224', 'resmlp_24_distilled_224']
    model = None
    for tm in names:
        if model_name in tm:
            if not tm.startswith('resnetv2'):
                raise NotImplementedError("only the ResNetV2-50x1-BiT path is implemented natively (got %s)" % tm)
            model = ResNetV2(num_classes=NUM_CLASSES_DICT[dataset_name], seed=seed)
            if not random_init:
                ck = os.path.join(model_dir, dataset_name, tm + '_cutout2_128_{}.pth'.format(dataset_name))
                checkpoint = torch.load(ck, map_location='cpu')
                model.load_state_dict(checkpoint['state_dict'])
    return model


class Normalize(object):
    """transforms.Normalize(mean, std) without the torchvision dependency."""

    def __init__(self, mean, std):
        self.mean, self.std = list(mean), list(std)

    def __call__(self, x):
        mean = torch.as_tensor(self.mean, dtype=x.dtype, device=x.device).view(-1, 1, 1)
        std = torch.as_tensor(self.std, dtype=x.dtype, device=x.device).view(-1, 1, 1)
        return (x - mean) / std

    def is_half_half(self):
        return all(m == 0.5 for m in self.mean) and all(s == 0.5 for s in self.std)


def get_normalize(dataset_name, model_name):
    return Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5])


class NormModel(torch.nn.Module):
    """utils.py:71-78.  When the wrapped model is the native ResNetV2 and the normalisation is
    the reference's (0.5, 0.5), the normalisation is fused into the K1 kernel.  There the logits are
    differentiable with respect to x when x requires grad (``ops.eot_logits``); the parameters get no gradient unless
    the model's ``param_grads_(True)`` is on."""

    def __init__(self, model, normalize):
        super(NormModel, self).__init__()
        self.model = model
        self.normalize = normalize

    def forward(self, x):
        if isinstance(self.model, ResNetV2) and isinstance(self.normalize, Normalize) and self.normalize.is_half_half():
            if torch.is_grad_enabled() and (x.requires_grad or self.model._param_grads):
                from .ops import eot_logits
                return eot_logits(self, x, param_grads=self.model._param_grads)
            return self.model.forward_unit(x)
        return self.model(self.normalize(x))


def unwrap_native(model):
    """DataParallel(NormModel(ResNetV2)) -> ResNetV2, else TypeError (no generic-module path:
    the hot loop exists only as native kernels for this architecture)."""
    m = model
    if isinstance(m, torch.nn.DataParallel):
        m = m.module
    if isinstance(m, NormModel):
        if not (isinstance(m.normalize, Normalize) and m.normalize.is_half_half()):
            raise TypeError("native DorPatch path needs NormModel with mean=std=0.5")
        m = m.model
    if not isinstance(m, ResNetV2):
        raise TypeError("native DorPatch path supports dorpatch_b200.ResNetV2 (resnetv2_50x1_bit) only, got %s"
                        % type(m).__name__)
    return m


class SyntheticImages(torch.utils.data.Dataset):
    """Deterministic synthetic [3,size,size] images in [0,1] (no dataset is reachable offline)."""

    def __init__(self, n, size=224, num_classes=1000, seed=0):
        self.n, self.size, self.num_classes, self.seed = n, size, num_classes, seed

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1000003 + i)
        return torch.rand(3, self.size, self.size, generator=g), int(torch.randint(0, self.num_classes, (1,), generator=g))


def get_dataset(dataset_name, data_dir='/home/data', train=False, batch_size=128, shuffle=True, synthetic=0,
                img_size=224):
    """utils.py:81-102; `synthetic=N` serves N synthetic images instead of torchvision data."""
    if synthetic:
        dataset = SyntheticImages(synthetic, img_size, NUM_CLASSES_DICT[dataset_name])
        print('Dataset has {} instances'.format(len(dataset)))
        return torch.utils.data.DataLoader(dataset, batch_size=batch_size, shuffle=shuffle, num_workers=0)
    import torchvision.transforms as transforms
    from torchvision import datasets
    dataset_dict = {'cifar10': datasets.CIFAR10, 'cifar100': datasets.CIFAR100, 'imagenet': datasets.ImageNet}
    args_dict = {'cifar10': {'train': train, 'download': True}, 'cifar100': {'train': train, 'download': True},
                 'imagenet': {'split': 'train' if train else 'val'}}
    size = 224
    dataset = dataset_dict[dataset_name](
        root=os.path.join(data_dir, dataset_name),
        transform=transforms.Compose([transforms.Resize(int(size / 0.875)), transforms.CenterCrop((size, size)),
                                      transforms.ToTensor()]),
        **args_dict[dataset_name])
    print('Dataset has {} instances'.format(len(dataset)))
    return torch.utils.data.DataLoader(dataset, batch_size=batch_size, shuffle=shuffle, num_workers=1, pin_memory=True)


def clip(mask, pattern, x, eps):
    """utils.py:105-110 on the native paste kernel: returns delta_x (caller adds x)."""
    if not x.is_cuda:
        raise RuntimeError("dorpatch_b200.utils.clip runs on the native CUDA engine only (no CPU fallback)")
    from .runtime import shared_engine
    eng = shared_engine(x.shape[-1], x.shape[0])
    x, mask, pattern = x.contiguous().float(), mask.contiguous().float(), pattern.contiguous().float()
    _, _, scale = eng.paste(x, mask, pattern, eps)       # the native kernel's min(eps / ||delta||_2, 1) per image
    # delta itself (utils.py:107-110), not (x + delta) - x: the latter loses delta's low bits to cancellation
    return mask * (pattern - x) * torch.from_numpy(scale).to(x.device).view(-1, 1, 1, 1)


def convert_float_list_to_str(l):
    return ', '.join(["%.2f" % i for i in l])
