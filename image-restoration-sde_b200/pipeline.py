"""Batched restoration front-end (SURVEY.md 8 f-2 / f-3): uint8 images in, uint8 images out.

The reference's ``test.py`` loops (codes/config/*/test.py:96-130) handle one image at a time: read_img ``/255.`` on the
CPU (codes/data/util.py:72), ``noise_state`` with the CPU generator (sde_utils.py:360-361, test.py:104), pageable H2D
of fp32 tensors, the chain, fp32 D2H, ``tensor2img`` on the CPU (img_utils.py:136-163).  Here the same work is staged
for a ~50-100 ms/image chain:

  uint8 HWC/BGR images --pinned H2D (3 B/px, side stream)--> img2tensor (device) --> [latent encode] -->
  noise_state (device Philox) --> reverse_{sde,ode,posterior} --> [latent decode] --> tensor2img (device)
  --D2H of uint8 (3 B/px)--> numpy images

Batches are assembled from same-sized images.  Every image carries a uid (its index in the input list + ``first_uid``)
and the device Philox is keyed by (seed, uid, t, element), so an image's result is bit-identical whether it is
restored alone, in any batch, or on any rank: batching keeps the reference's single-image semantics.
"""
import numpy as np
import torch

from . import imaging


def plan_batches(shapes, batch_size):
    """Group image indices by shape (first-seen order), then cut each group into batches of <= batch_size.
    Pure host logic: ``shapes`` is a list of hashable (H, W, C)."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    groups = {}
    for i, s in enumerate(shapes):
        groups.setdefault(tuple(s), []).append(i)
    out = []
    for s, idx in groups.items():
        for k in range(0, len(idx), batch_size):
            out.append((s, idx[k:k + batch_size]))
    return out


class Restorer:
    """``Restorer(sde, mode="sde", batch_size=8, seed=0, T=-1, autoencoder=None).restore(images)``.

    ``sde`` is an :class:`irsde_b200.IRSDE` with ``set_model`` done.  ``autoencoder`` (an :class:`irsde_b200.UNet`)
    switches to the Refusion latent path (encode -> latent chain -> decode, latent-dehazing/test.py:88-96)."""

    def __init__(self, sde, mode="sde", batch_size=8, seed=0, T=-1, autoencoder=None, device=None):
        if mode not in ("sde", "ode", "posterior"):
            raise ValueError("mode must be 'sde', 'ode' or 'posterior'")
        self.sde, self.mode, self.batch_size, self.seed, self.T, self.ae = sde, mode, int(batch_size), int(seed), T, autoencoder
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._copy = None
        self._pin_in, self._pin_out = {}, {}

    def _pinned(self, pool, shape):
        buf = pool.get(shape)
        if buf is None:
            buf = torch.empty(shape, dtype=torch.uint8).pin_memory()
            pool[shape] = buf
        return buf

    def _stage_in(self, images, idx, shape):
        """Pack the batch into pinned memory and start its H2D copy on the side stream."""
        H, W, C = shape
        pin = self._pinned(self._pin_in, (self.batch_size, H, W, C))
        for k, i in enumerate(idx):
            pin[k].copy_(torch.from_numpy(np.ascontiguousarray(images[i])))
        with torch.cuda.stream(self._copy):
            dev = pin[:len(idx)].to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._copy)
        return dev, ev

    @torch.no_grad()
    def restore_batch(self, lq_u8, uids):
        """uint8 CUDA tensor [B,H,W,C] (BGR) + uids -> uint8 CUDA tensor [B,H,W,C] (BGR)."""
        sde = self.sde
        saved = (sde.rng, sde.seed, sde.seed_auto_increment, sde.image_uids)
        sde.rng, sde.seed, sde.seed_auto_increment, sde.image_uids = "philox", self.seed, False, list(uids)
        try:
            lq = imaging.img2tensor_device(lq_u8)
            skips = None
            if self.ae is not None:
                lq, skips = self.ae.encode(lq)
            sde.set_mu(lq)
            xT = sde.noise_state(lq)
            run = {"sde": sde.reverse_sde, "ode": sde.reverse_ode, "posterior": sde.reverse_posterior}[self.mode]
            x0 = run(xT, T=self.T)
            if self.ae is not None:
                x0 = self.ae.decode(x0, skips)
            return imaging.tensor2img_device(x0)
        finally:
            sde.rng, sde.seed, sde.seed_auto_increment, sde.image_uids = saved

    def restore(self, images, first_uid=0):
        """List of uint8 [H,W,3] (BGR, the cv2 order) numpy images -> list of restored uint8 images, same order."""
        for im in images:
            if not (isinstance(im, np.ndarray) and im.dtype == np.uint8 and im.ndim == 3):
                raise TypeError("images must be uint8 numpy arrays [H,W,C]")
        if not torch.cuda.is_available():
            raise RuntimeError("irsde_b200.Restorer runs on CUDA (sm_90a) only; there is no CPU path")
        batches = plan_batches([im.shape for im in images], self.batch_size)
        out = [None] * len(images)
        with torch.cuda.device(self.device):
            if self._copy is None:
                self._copy = torch.cuda.Stream(self.device)
            main = torch.cuda.current_stream()
            staged = self._stage_in(images, batches[0][1], batches[0][0]) if batches else None
            pending = None   # (pinned result, event, indices) of the previous batch
            for k, (shape, idx) in enumerate(batches):
                dev, ev = staged
                main.wait_event(ev)
                res = self.restore_batch(dev, [first_uid + i for i in idx])
                done = torch.cuda.Event()
                done.record(main)
                # the next batch's upload overlaps this batch's chain; its pinned buffer is free once `ev` fired
                if k + 1 < len(batches):
                    ev.synchronize()
                    staged = self._stage_in(images, batches[k + 1][1], batches[k + 1][0])
                if pending is not None:
                    self._collect(pending, out)
                H, W, C = shape
                pin = self._pinned(self._pin_out, (self.batch_size, H, W, C))
                with torch.cuda.stream(self._copy):
                    self._copy.wait_event(done)
                    pin[:len(idx)].copy_(res, non_blocking=True)
                    cev = torch.cuda.Event()
                    cev.record(self._copy)
                res.record_stream(self._copy)
                pending = (pin, cev, idx)
            if pending is not None:
                self._collect(pending, out)
        return out

    @staticmethod
    def _collect(pending, out):
        pin, ev, idx = pending
        ev.synchronize()
        for k, i in enumerate(idx):
            out[i] = pin[k].numpy().copy()
