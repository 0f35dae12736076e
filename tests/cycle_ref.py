"""TEST INFRASTRUCTURE — CPU restatement of the reference trainer's masking and cycle augmentation
(``src/smirk_trainer.py``: step1 masking :76-92, step2 augmentation :189-248, step2 masking :262-293).

Every random draw is an explicit input, named as the device stages export them (``TrainMaskingStage(debug=True)``,
``CycleAugmentation(debug=True)``).  ``augment_draws_ref`` / ``sample_draws_ref`` / ``noise_draws_ref`` make those draws
from torch's global generator and Python's ``random`` in the reference's own order (``randperm`` first, then line by
line, left operand first), so under the same seeds these functions reproduce the reference step bit for bit; fed the
device's exported draws, they are what the device must equal bit for bit.  The masking is composed from
``oracle/masking_ref.py``.
"""
import random

import torch

from oracle import masking_ref


def group_bounds(R):
    return [0, R // 4, 2 * R // 4, 3 * R // 4, R]


# ------------------------------------------------------------------------------------------------- augmentation
def augment_draws_ref(R, E, De, templates, use_eyelids=True):
    """The augmentation's draws for Ke*B = R rows, from torch's global RNG and Python's ``random``, in the reference's
    order.  Template picks are (index into ``list(templates)``, row)."""
    c = group_bounds(R)
    n0, n1, n2, n3 = (c[i + 1] - c[i] for i in range(4))
    d = {"gids": torch.randperm(R)}                                                   # :200
    d["param_mask"] = torch.bernoulli(torch.ones((n0, E)) * 0.5)                     # :208
    d["randn0a"] = torch.randn((n0, E))                                               # :210, left to right
    d["rand0a"] = torch.rand((n0, 1))
    d["rand0b"] = torch.rand((n0, 1))                                                 # :211
    d["randn0b"] = torch.randn((n0, E))
    d["rand1a"] = torch.rand((n1, 1))                                                 # :215
    d["perm1"] = torch.randperm(n1)
    d["rand1b"] = torch.rand((n1, 1))
    d["randn1"] = torch.randn((n1, E))
    keys, picks, rows, u = list(templates.keys()), [], [], []
    for _ in range(n2):                                                               # :220-222, base_trainer.py:69-74
        k = random.choice(keys)
        r = random.randint(0, templates[k].shape[0] - 1)
        picks.append(keys.index(k)); rows.append(r)
        u.append(torch.rand((1, 1)))
    d["tmpl_key"], d["tmpl_row"] = torch.tensor(picks, dtype=torch.int64), torch.tensor(rows, dtype=torch.int64)
    d["rand2a"] = torch.cat(u, 0) if u else torch.zeros(0, 1)
    d["rand2b"] = torch.rand((n2, 1))                                                 # :223
    d["randn2"] = torch.randn((n2, E))
    d["jaw_mask"] = torch.bernoulli(torch.ones(R) * 0.5)                             # :226
    d["randn_jaw"] = torch.randn((R, 3))                                              # :227
    if use_eyelids:
        d["rand_eyelid"] = torch.rand(size=(R, De))                                   # :232
    d["rand3"] = torch.rand((n3, 1))                                                  # :239
    d["randn3"] = torch.randn((n3, E))
    d["rand3_eyelid"] = torch.rand(size=(n3, De))                                     # :242
    return d


def augment_ref(encoder_output, Ke, d, templates, num_expression=50, use_eyelids=True):
    """smirk_trainer.py:194-248 with the draws ``d`` given; fp32 on the CPU, op for op."""
    flame_feats = {}
    for k, v in encoder_output.items():
        tmp = v.clone().detach()
        flame_feats[k] = torch.cat(Ke * [tmp], dim=0)
    R = flame_feats["expression_params"].shape[0]
    c, gids = group_bounds(R), d["gids"]
    gids = [gids[c[0]:c[1]], gids[c[1]:c[2]], gids[c[2]:c[3]], gids[c[3]:c[4]]]
    new_expressions = d["randn0a"] * (1 + 2 * d["rand0a"]) * d["param_mask"] + flame_feats["expression_params"][gids[0]]
    flame_feats["expression_params"][gids[0]] = torch.clamp(new_expressions, -4.0, 4.0) + (0 + 0.2 * d["rand0b"]) * d["randn0b"]
    flame_feats["expression_params"][gids[1]] = (0.25 + 1.25 * d["rand1a"]) * flame_feats["expression_params"][gids[1]][d["perm1"]] + \
        (0 + 0.2 * d["rand1b"]) * d["randn1"]
    keys = list(templates.keys())
    for i in range(len(gids[2])):
        expression = templates[keys[int(d["tmpl_key"][i])]][int(d["tmpl_row"][i])][:num_expression]
        flame_feats["expression_params"][gids[2][i], :num_expression] = (0.25 + 1.25 * d["rand2a"][i:i + 1].view(1, 1)) * \
            torch.Tensor(expression).to(d["rand2a"].device)
    flame_feats["expression_params"][gids[2]] += (0 + 0.2 * d["rand2b"]) * d["randn2"]
    scale_mask = torch.Tensor([1, .1, .1]).to(d["jaw_mask"].device).view(1, 3) * d["jaw_mask"].view(-1, 1)
    flame_feats["jaw_params"] = flame_feats["jaw_params"] + d["randn_jaw"] * 0.2 * scale_mask
    flame_feats["jaw_params"][..., 0] = torch.clamp(flame_feats["jaw_params"][..., 0], 0.0, 0.5)
    if use_eyelids:
        flame_feats["eyelid_params"] += (-1 + 2 * d["rand_eyelid"]) * 0.25
        flame_feats["eyelid_params"] = torch.clamp(flame_feats["eyelid_params"], 0.0, 1.0)
    flame_feats["expression_params"][gids[3]] *= 0.0
    flame_feats["expression_params"][gids[3]] += (0 + 0.2 * d["rand3"]) * d["randn3"]
    flame_feats["jaw_params"][gids[3]] *= 0.0
    flame_feats["eyelid_params"][gids[3]] = d["rand3_eyelid"]
    return {k: v.detach() for k, v in flame_feats.items()}


# ------------------------------------------------------------------------------------------------- masking
def sample_draws_ref(tv, faces, base_prob, N):
    """masking.py:146-165: multinomial face indices and reflected barycentrics, from torch's global RNG."""
    B = tv.shape[0]
    w = masking_ref.face_probabilities_ref(tv, faces, base_prob)
    fidx = torch.multinomial(w, N, replacement=True)
    u, v = torch.rand(B * N), torch.rand(B * N)
    out = u + v > 1
    u[out], v[out] = 1 - u[out], 1 - v[out]
    return fidx, torch.stack((1 - (u + v), u, v), dim=1).view(B, N, 3)


def noise_draws_ref(R, S, random_mask):
    """masking.py:86-93: the noise multiplier and the patch centres, from torch's global RNG."""
    noise = torch.randn((R, 3, S, S)) * 0.05 + 1
    centres = torch.bernoulli(torch.ones((R, 1, S, S)) * random_mask) if random_mask > 0 else None
    return noise, centres


def transfer_pixels_ref(img, points1, points2):
    """masking.py:116-129 without rbound, vectorised: with duplicate targets the last pair in index order wins."""
    R, C, H, W = img.shape
    N = points1.shape[1]
    tgt = (torch.arange(R).view(-1, 1) * H + points2[..., 1]) * W + points2[..., 0]
    win = torch.full((R * H * W,), -1, dtype=torch.int64)
    win = win.scatter_reduce(0, tgt.reshape(-1), torch.arange(N).repeat(R), "amax")
    win = win.view(R, H * W)
    j = win.clamp(min=0)
    src = points1[..., 1].gather(1, j) * W + points1[..., 0].gather(1, j)
    out = img.reshape(R, C, H * W).gather(2, src[:, None].expand(-1, C, -1))
    return torch.where((win >= 0)[:, None], out, torch.zeros_like(out)).view(R, C, H, W)


def conflicting_targets(points1, points2, size=224):
    """[R,1,S,S] bool: target pixels that two or more pairs with different source pixels write.  There the reference's
    CPU ``transfer_pixels`` keeps whichever pair its indexed assignment happens to store last (an implementation detail of
    torch's index_put, neither the first nor the last pair in index order); the device keeps the last pair."""
    R, N = points2.shape[:2]
    tgt = (points2[..., 1] * size + points2[..., 0]).reshape(R, N)
    src = (points1[..., 1] * size + points1[..., 0]).reshape(R, N)
    out = torch.zeros(R, size * size, dtype=torch.bool)
    for r in range(R):
        pairs = torch.unique(torch.stack((tgt[r], src[r]), 1), dim=0)
        t, n = torch.unique(pairs[:, 0], return_counts=True)
        out[r, t[n > 1]] = True
    return out.view(R, 1, size, size)


def rendered_mask_first(rendered):
    return 1 - (rendered == 0).all(dim=1, keepdim=True).float()                       # smirk_trainer.py:77


def rendered_mask_second(rendered):
    return (rendered > 0).all(dim=1, keepdim=True).float()                            # smirk_trainer.py:290


def first_path_ref(img, hull, tv, rendered, faces, fidx, bary, noise, centres, wr=10, image_size=224, points=None):
    """smirk_trainer.py:76-92 given the draws -> (masked_img, npoints); ``points`` replaces the computed npoints."""
    npoints = masking_ref.points_from_coords_ref(tv, faces, fidx, bary, image_size)[..., :2] if points is None else points
    extra_points = transfer_pixels_ref(img, npoints, npoints)
    return masking_ref.masking_ref(img, hull, extra_points, wr, rendered_mask=rendered_mask_first(rendered), noise_mult=noise,
                                   random_centres=centres), npoints


def second_path_ref(img, hull, tv, tv2, rendered2, faces, fidx, bary, Ke, noise, centres, wr=10, image_size=224, points1=None, points2=None):
    """smirk_trainer.py:268-293 given the draws -> (masked_img_2nd_path, points1, points2)."""
    if points1 is None:
        points1 = masking_ref.points_from_coords_ref(tv, faces, fidx, bary, image_size)[..., :2]
    if points2 is None:
        points2 = masking_ref.points_from_coords_ref(tv2, faces, fidx.repeat(Ke, 1), bary.repeat(Ke, 1, 1), image_size)[..., :2]
    extra_points = transfer_pixels_ref(img.repeat(Ke, 1, 1, 1), points1.repeat(Ke, 1, 1), points2)
    masked = masking_ref.masking_ref(img.repeat(Ke, 1, 1, 1), hull.repeat(Ke, 1, 1, 1), extra_points, wr,
                                     rendered_mask=rendered_mask_second(rendered2), noise_mult=noise, random_centres=centres)
    return masked, points1, points2
