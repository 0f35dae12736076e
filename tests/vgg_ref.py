"""TEST ORACLE — the reference's VGGPerceptualLoss (src/losses/VGGPerceptualLoss.py) restated in torch ops over a
``state_dict`` of smirk_b200.VGGPerceptualLoss, and a replay variant.

``vgg_loss_ref(sd, x, y)``: x, y [B,3,224,224] -> the loss (the reference's bilinear resize to 224^2 is the identity there).

``vgg_loss_replay_ref(sd, x, y, saved)`` runs the same arithmetic with the discrete choices taken from a device run's
``saved_activations``: every ReLU as z * [saved > 0], every max pool as a gather at the first maximum of the device's saved
pool input, and every L1 term as sum(s * (phi(x) - phi(y))) / N with the device's sign maps s.  Its forward equals the loss
wherever the device agrees with it, and autograd through it is the exact backward of the device's own choices, the
oracle of the device's input gradient.
"""
import torch
import torch.nn.functional as F

CONVS = ["blocks.0.0", "blocks.0.2", "blocks.1.5", "blocks.1.7", "blocks.2.10", "blocks.2.12", "blocks.2.14",
         "blocks.3.17", "blocks.3.19", "blocks.3.21"]
NAMES = ["relu1_1", "relu1_2", "relu2_1", "relu2_2", "relu3_1", "relu3_2", "relu3_3", "relu4_1", "relu4_2", "relu4_3"]
TAP_CONVS = [1, 3, 6, 9]
SIGNS = ["sign1_2", "sign2_2", "sign3_3", "sign4_3"]
POOL_AFTER = {1, 3, 6}                     # a 2x2 max pool follows these convs


def vgg_state_dict(template, seed=7):
    """Seeded weights for a VGGPerceptualLoss ``state_dict`` template: He-scaled convs (activations stay O(1) through ten
    layers) from synth_inputs.random_state_dict, the reference's mean / std buffers kept."""
    from smirk_b200 import synth_inputs
    sd = synth_inputs.random_state_dict(template, seed=seed)
    sd["mean"], sd["std"] = template["mean"].clone(), template["std"].clone()
    return sd


def normalise(sd, v):
    return (v * 0.5 + 0.5 - sd["mean"]) / sd["std"]


def activations(sd, v):
    """The ten post-ReLU outputs of features[:23] on the normalised input v."""
    out = []
    for l, k in enumerate(CONVS):
        v = F.relu(F.conv2d(v, sd[k + ".weight"], sd[k + ".bias"], padding=1))
        out.append(v)
        if l in POOL_AFTER:
            v = F.max_pool2d(v, 2, 2)
    return out


def vgg_loss_ref(sd, x, y):
    ax, ay = activations(sd, normalise(sd, x)), activations(sd, normalise(sd, y))
    loss = 0.0
    for l in TAP_CONVS:
        loss = loss + F.l1_loss(ax[l], ay[l])
    return loss


def _pool_at(v, at):
    """2x2 max pool of v taken at the first maximum (row-major) of each window of `at`."""
    B, C, S, _ = v.shape
    win = lambda t: t.reshape(B, C, S // 2, 2, S // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, S // 2, S // 2, 4)
    idx = torch.argmax(win(at), dim=-1, keepdim=True)            # first occurrence of the maximum
    return torch.gather(win(v), -1, idx).squeeze(-1)


def replay_activations(sd, v, saved_half):
    """activations() with the ReLU masks and pool indices of `saved_half` ({relu name: [B,C,H,W]})."""
    out = []
    for l, k in enumerate(CONVS):
        z = F.conv2d(v, sd[k + ".weight"], sd[k + ".bias"], padding=1)
        v = z * (saved_half[NAMES[l]] > 0).to(z.dtype)
        out.append(v)
        if l in POOL_AFTER:
            v = _pool_at(v, saved_half[NAMES[l]])
    return out


def vgg_loss_replay_ref(sd, x, y, saved, record=None):
    """saved: {"relu*": [2B,C,H,W] (x's images, then y's), "sign*": [B,C,H,W]} as VGGPerceptualLoss.saved_activations.
    record (optional list): receives the tensors of the graph a gradient passes through, x's normalised input and ten
    post-ReLU outputs, then y's."""
    B = x.shape[0]
    nx, ny = normalise(sd, x), normalise(sd, y)
    ax = replay_activations(sd, nx, {k: saved[k][:B] for k in NAMES})
    ay = replay_activations(sd, ny, {k: saved[k][B:] for k in NAMES})
    if record is not None:
        record += [nx] + ax + [ny] + ay
    loss = 0.0
    for t, l in enumerate(TAP_CONVS):
        s = saved[SIGNS[t]].to(ax[l].dtype)
        loss = loss + (s * (ax[l] - ay[l])).sum() / ax[l].numel()
    return loss


CHANNELS = [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512), (512, 512)]


def integer_state_dict(seed):
    """A VGGPerceptualLoss state_dict on which every quantity of the forward and the input gradient is a small multiple
    of 0.5 (tests/test_vgg_loss_layers_host.py checks it): output channel co of each conv has weight +1 on input channel
    co mod cin at a random tap and -1 at a random other (channel, tap), all other weights 0; biases in {0, 1}; mean and
    std distinct per channel (a channel mix-up in the normalisation shows) and such that the normalised input of
    integer_inputs is a multiple of 0.5 in [-3, 3]."""
    g = torch.Generator().manual_seed(seed)
    sd = {"mean": torch.tensor([0.5, 0.25, 0.75]).view(1, 3, 1, 1), "std": torch.tensor([0.5, 0.25, 0.25]).view(1, 3, 1, 1)}
    for k, (cin, cout) in zip(CONVS, CHANNELS):
        w = torch.zeros(cout, cin * 9)
        co = torch.arange(cout)
        plus = (co % cin) * 9 + torch.randint(0, 9, (cout,), generator=g)
        minus = (plus + torch.randint(1, cin * 9, (cout,), generator=g)) % (cin * 9)       # any other (channel, tap)
        w[co, plus], w[co, minus] = 1.0, -1.0
        sd[k + ".weight"] = w.view(cout, cin, 3, 3)
        sd[k + ".bias"] = torch.randint(0, 2, (cout,), generator=g).float()
    return sd


def integer_inputs(B, seed):
    """x, y [B,3,224,224] in {-1, -0.5, 0, 0.5, 1}; y is x with 30 % of its entries drawn again."""
    g = torch.Generator().manual_seed(seed)
    draw = lambda: torch.randint(-2, 3, (B, 3, 224, 224), generator=g).float() * 0.5
    x = draw()
    y = torch.where(torch.rand(B, 3, 224, 224, generator=g) < 0.3, draw(), x)
    return x, y


def integer_upstream(B):
    """The loss's upstream gradient B * 224^2 * 64: tap t's L1 gradient g / numel_t is then exactly 2^t."""
    return float(B * 224 * 224 * 64)


def oracle_saved(sd, x, y):
    """The oracle's own activations and sign maps, in the layout of saved_activations (for testing the replay)."""
    with torch.no_grad():
        ax, ay = activations(sd, normalise(sd, x)), activations(sd, normalise(sd, y))
    out = {NAMES[l]: torch.cat([ax[l], ay[l]]) for l in range(len(CONVS))}
    for t, l in enumerate(TAP_CONVS):
        out[SIGNS[t]] = torch.sign(ax[l] - ay[l]).to(torch.int8)
    return out
