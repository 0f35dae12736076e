"""TEST INFRASTRUCTURE — config_train's step (``src/smirk_trainer.py``: ``step1`` :35-179, ``step2`` :184-332, ``step``
:348-392) on the device, through the drop-in classes and the two device stages (``TrainMaskingStage``,
``CycleAugmentation``), with config_train.yaml's loss weights (landmarks 100, L1 10, VGG 10, emotion 0, expression
regularisation 1e-3, jaw 1e-2, cycle 1; ``optimize_expression`` on, ``optimize_shape`` off, no base model, Ke = 1,
``use_eyelids`` on).  Each path is one function from its inputs to its loss and the gradients of the parameters it
trains, so a path can be captured in one CUDA graph.

The reference's host-syncing lines, and what replaces each:
  * ``0 if torch.sum(valid_landmarks) == 0 else F.mse_loss(lmk[valid, :17], gt[valid, :17])`` (:64, a host branch on a
    device sum, then boolean indexing): the squared error weighted by the flags, summed, over
    ``max(1, 17 * 2 * sum(flags))`` — the same mean where a face is valid, 0 where none is; summed in another order.
  * ``value.item()`` of every loss (:156-157, :319-320): the losses stay device tensors.
  * ``outputs[key].detach().cpu()`` (:174-175) and the ``visualize_every`` stacks (:326-330), with the second
    FLAME + Renderer pass of the reconstruction they alone read (:302-303): dropped; they do not enter a loss.
  * ``masking_utils.mesh_based_mask_uniform_faces`` / ``transfer_pixels`` / ``masking`` (:76-92, :262-293;
    ``torch.multinomial``, boolean indexing in ``random_barycentric``): ``TrainMaskingStage.first_path`` / ``second_path``.
  * the augmentation's ``torch.randperm`` on the host, the Python ``random`` template loop with one host-to-device copy per
    row and ~30 small launches (:189-248): ``CycleAugmentation``.
The freeze schedule is ``set_freeze_status`` (base_trainer.py:258-268) with the batch index's parity: even = encoder
frozen in the second path, odd = generator frozen (``utils.freeze_module``: eval, ``requires_grad_(False)``) and its
reconstruction detached.  The whole encoder runs in one mode per call: the drop-in encoder runs its three backbones in
one launch sequence, so the reference's split (only the expression encoder unfrozen after ``unfreeze_encoder``) is not
restated; every encoder parameter gets its gradient.
"""
import copy

import numpy as np
import torch
import torch.nn.functional as F

import make_golden_cycle as mgc

DEV = "cuda:0"
W = dict(landmark_loss=100.0, perceptual_vgg_loss=10.0, reconstruction_loss=10.0, expression_regularization=1e-3,
         jaw_regularization=1e-2, cycle_loss=1.0)
GEN_CFG = (6, 3, 32, 5)


def make_bases(asset_root):
    """Shared modules of the flow: encoder and generator weights (random_state_dict, seed 7), FLAME, Renderer, the VGG loss
    with the weights of its golden file, the mesh faces and face probabilities."""
    import smirk_b200
    import make_golden_vgg_loss as mv
    from oracle import flame_ref
    from smirk_b200 import synth_inputs
    enc = smirk_b200.SmirkEncoder()
    enc.load_state_dict(synth_inputs.random_state_dict(enc.state_dict(), seed=7))
    gen = smirk_b200.SmirkGenerator(*GEN_CFG)
    gen.load_state_dict(synth_inputs.random_state_dict(gen.state_dict(), seed=7))
    vgg = smirk_b200.VGGPerceptualLoss(weights=None)
    vgg.load_state_dict(mv.golden_state_dict())
    g = np.load(mgc.MASKING)
    return dict(enc=enc, gen=gen, fl=smirk_b200.FLAME().to(DEV), rd=smirk_b200.Renderer().to(DEV), vgg=vgg.to(DEV),
                faces=flame_ref.FlameConstants(asset_root).faces_tensor, base_prob=torch.from_numpy(g["base_prob"]))


def make_batch(B, seed):
    """One batch on the device: images, hull masks, FAN (with some faces flagged invalid) and mediapipe landmarks."""
    from smirk_b200 import synth_inputs
    g = np.load(mgc.MASKING)
    gen = torch.Generator().manual_seed(seed)
    flags = torch.rand(B, generator=gen) > 0.25
    return {"img": synth_inputs.images(B, seed).to(DEV),
            "mask": torch.from_numpy(g["hull"]).float()[torch.arange(B) % 2].to(DEV),
            "landmarks_fan": (torch.rand(B, 68, 2, generator=gen) - 0.5).to(DEV),
            "landmarks_mp": (torch.rand(B, 105, 2, generator=gen) - 0.5).to(DEV),
            "flag_landmarks_fan": flags.to(DEV)}


class TrainFlow:
    """Train-mode encoder and generator at one precision, the shared frozen modules, and the two device stages."""

    def __init__(self, bases, precision=3, seed=0):
        from smirk_b200.cycle import CycleAugmentation
        from smirk_b200.masking import TrainMaskingStage
        self.enc = copy.deepcopy(bases["enc"]).to(DEV).train().allow_train_mode_(True)
        for m in self.enc.modules():
            if hasattr(m, "precision"):
                m.precision = precision
        self.gen = copy.deepcopy(bases["gen"]).to(DEV).train().allow_train_mode_(True)
        self.gen.precision = precision
        self.fl, self.rd, self.vgg = bases["fl"], bases["rd"], bases["vgg"]
        self.masking = TrainMaskingStage(bases["faces"], bases["base_prob"], mask_ratio=0.01, mask_dilation_radius=10, seed=seed)
        self.augment = CycleAugmentation(mgc.synthetic_templates(), num_expression=50, use_eyelids=True, seed=seed + 1)
        self.seed = seed

    def reseed(self, counter):
        self.masking.reseed(self.seed, counter)
        self.augment.reseed(self.seed + 1, counter)

    def stats(self):
        return [v for m in (self.enc, self.gen) for k, v in m.state_dict().items() if "running_" in k or "num_batches" in k]

    def params1(self):
        return list(self.enc.parameters()) + list(self.gen.parameters())

    def params2(self, parity):
        return list(self.gen.parameters()) if parity % 2 == 0 else list(self.enc.parameters())

    # ---- step1 (smirk_trainer.py:35-154) -> (loss_first_path, encoder_output)
    def step1(self, batch):
        img = batch["img"]
        B = img.shape[0]
        encoder_output = self.enc(img)
        fo = self.fl(encoder_output)
        ro = self.rd(fo["vertices"], encoder_output["cam"], landmarks_fan=fo["landmarks_fan"], landmarks_mp=fo["landmarks_mp"])
        rendered_img = ro["rendered_img"]
        w = batch["flag_landmarks_fan"].float()
        d = (ro["landmarks_fan"][:, :17, :2] - batch["landmarks_fan"][:, :17]) ** 2
        landmark_loss_fan = (d * w[:, None, None]).sum() / (w.sum() * 34).clamp(min=1.0)
        landmark_loss_mp = F.mse_loss(ro["landmarks_mp"][..., :2], batch["landmarks_mp"])
        zeros = {k: torch.zeros(B, n, device=img.device) for k, n in (("expression_params", 50), ("jaw_params", 3))}
        expression_regularization = torch.mean((encoder_output["expression_params"] - zeros["expression_params"]) ** 2)
        jaw_regularization = torch.mean((encoder_output["jaw_params"] - zeros["jaw_params"]) ** 2)
        masked_img = self.masking.first_path(img, batch["mask"], ro["transformed_vertices"], rendered_img)
        reconstructed_img = self.gen(torch.cat([rendered_img, masked_img], dim=1))
        reconstruction_loss = F.l1_loss(reconstructed_img, img, reduction="none").mean()
        perceptual_vgg_loss = self.vgg(reconstructed_img, img)
        loss = (expression_regularization * W["expression_regularization"] + jaw_regularization * W["jaw_regularization"]) + \
            (landmark_loss_fan * W["landmark_loss"] + landmark_loss_mp * W["landmark_loss"]) + \
            (perceptual_vgg_loss * W["perceptual_vgg_loss"] + reconstruction_loss * W["reconstruction_loss"])
        return loss, encoder_output

    # ---- step2 (smirk_trainer.py:184-317) -> loss_second_path; the caller has applied the freeze status
    def step2(self, encoder_output, batch, parity):
        freeze_generator = parity % 2 == 1
        img, masks = batch["img"], batch["mask"]
        Ke = 1
        flame_feats = self.augment(encoder_output, Ke=Ke)
        with torch.no_grad():
            fo = self.fl(encoder_output)
            ro = self.rd(fo["vertices"], encoder_output["cam"])
            fo2 = self.fl(flame_feats)
            ro2 = self.rd(fo2["vertices"], encoder_output["cam"])
            rendered_img_2nd_path = ro2["rendered_img"].detach()
            masked = self.masking.second_path(img, masks, ro["transformed_vertices"], ro2["transformed_vertices"],
                                              rendered_img_2nd_path, Ke=Ke)
        reconstructed = self.gen(torch.cat([rendered_img_2nd_path, masked], dim=1).detach())
        if freeze_generator:
            reconstructed = reconstructed.detach()
        recon_feats = self.enc(reconstructed)
        cycle_loss = 1.0 * F.mse_loss(recon_feats["expression_params"], flame_feats["expression_params"]) + \
            10.0 * F.mse_loss(recon_feats["jaw_params"], flame_feats["jaw_params"])
        cycle_loss = cycle_loss + 10.0 * F.mse_loss(recon_feats["eyelid_params"], flame_feats["eyelid_params"])
        if not freeze_generator:
            cycle_loss = cycle_loss + 1.0 * F.mse_loss(recon_feats["shape_params"], flame_feats["shape_params"])
        return cycle_loss * W["cycle_loss"]

    def set_freeze(self, parity):
        """base_trainer.set_freeze_status for a batch index of this parity, applied as step() applies it."""
        if parity % 2 == 0:
            self.enc.eval().requires_grad_(False)
        else:
            self.gen.eval().requires_grad_(False)

    def unfreeze(self):
        self.enc.train().requires_grad_(True)
        self.gen.train().requires_grad_(True)

    # ---- one path as a function of its inputs: (loss, gradients of the parameters it trains; None where a parameter does
    # not reach the loss, e.g. the pose backbone in a second path whose loss reads no pose)
    def path1(self, batch):
        loss, encoder_output = self.step1(batch)
        grads = torch.autograd.grad(loss, self.params1(), allow_unused=True)
        return loss.detach(), grads, {k: v.detach() for k, v in encoder_output.items()}

    def path2(self, encoder_output, batch, parity):
        params = self.params2(parity)
        self.set_freeze(parity)
        try:
            loss = self.step2(encoder_output, batch, parity)
            grads = torch.autograd.grad(loss, params, allow_unused=True)
        finally:
            self.unfreeze()
        return loss.detach(), grads
