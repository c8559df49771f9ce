"""Offline pre-encode wire format: tokenise once, train from token shards (SURVEY.md 8f-3).

Reference writer: scripts/pre_encode.py:136-243 -- one webdataset tar per source shard; per sample the members
``<key>.<vae checkpoint with '/' -> '.'>.pth`` (image token ids, ``torch.save``d LongTensor [L]),
``<key>.<text-encoder checkpoint>.pth`` (encoder hidden states [77, E]) and ``<key>.json`` (metadata incl.
``attention_mask_length``).  Reference reader: training/data.py:561-573 -- members decoded with ``torch.load``
(webdataset ``torch_loads``), the extension lower-cased by webdataset's key grouping, renamed to ``image_input_ids`` /
``encoder_hidden_states``; consumed by training/train_muse.py:689-690.

webdataset is not in this image, and the format is plain POSIX tar, so writer and reader are implemented on ``tarfile``
with webdataset's member conventions (basename split at the FIRST dot into key and extension, all members of a sample
contiguous, mode 0444, owner "bigdata").  The tokeniser in front is this package's ``VQGANModel`` / ``MaskGitVQGAN``
``get_code`` (wgmma convolutions + bit-exact arg-min); ``pre_encode_images`` overlaps the device->host copy of one
batch with the encode of the next."""
from __future__ import annotations

import io
import json
import re
import tarfile
import time
from typing import Dict, Iterable, Iterator, Optional

import torch


def checkpoint_ext(checkpoint: str) -> str:
    """``openMUSE/vqgan-f16-8192-laion`` -> ``openMUSE.vqgan-f16-8192-laion.pth`` (scripts/pre_encode.py:54-56)."""
    return ".".join(checkpoint.split("/")) + ".pth"


def _torch_bytes(t: torch.Tensor) -> bytes:
    buf = io.BytesIO()
    torch.save(t, buf)  # webdataset's default encoder for the "pth" extension
    return buf.getvalue()


class PreEncodedShardWriter:
    """Writes one pre-encoded shard.  ``dest`` is a path or a binary file object (e.g. the stdin of an upload pipe)."""

    def __init__(self, dest, vae_checkpoint: str, text_encoder_checkpoint: Optional[str] = None, mtime: Optional[float] = None):
        self.tar = tarfile.open(dest, "w") if isinstance(dest, str) else tarfile.open(fileobj=dest, mode="w|")
        self.vae_ext = checkpoint_ext(vae_checkpoint)
        self.text_ext = None if text_encoder_checkpoint is None else checkpoint_ext(text_encoder_checkpoint)
        self.mtime = mtime
        self.count = 0

    def _add(self, name: str, data: bytes):
        ti = tarfile.TarInfo(name)
        ti.size = len(data)
        ti.mtime = time.time() if self.mtime is None else self.mtime
        ti.mode = 0o444
        ti.uname = ti.gname = "bigdata"
        self.tar.addfile(ti, io.BytesIO(data))

    def write(self, key: str, image_tokens: torch.Tensor, encoder_hidden_states: Optional[torch.Tensor] = None,
              metadata: Optional[dict] = None, extra: Optional[Dict[str, torch.Tensor]] = None):
        if "." in key.rsplit("/", 1)[-1]:
            raise ValueError(f"sample key {key!r}: the basename must not contain '.', webdataset splits key and extension at the first dot")
        if image_tokens.dtype != torch.int64:
            raise TypeError("image token ids are stored as int64 (what get_code returns and nn.Embedding consumes)")
        self._add(f"{key}.{self.vae_ext}", _torch_bytes(image_tokens.detach().cpu().clone()))
        for ext, t in (extra or {}).items():  # e.g. a second tokenizer's ids (the reference stores f8 and f16 codes)
            self._add(f"{key}.{checkpoint_ext(ext)}", _torch_bytes(t.detach().cpu().clone()))
        if encoder_hidden_states is not None:
            if self.text_ext is None:
                raise ValueError("writer was opened without a text_encoder_checkpoint")
            self._add(f"{key}.{self.text_ext}", _torch_bytes(encoder_hidden_states.detach().cpu().clone()))
        if metadata is not None:
            self._add(f"{key}.json", json.dumps(metadata).encode("utf-8"))
        self.count += 1

    def close(self):
        self.tar.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False


_SPLIT = re.compile(r"^((?:.*/|)[^.]+)[.]([^/]*)$")  # webdataset's base_plus_ext


def iter_pre_encoded(src, vae_checkpoint: str, text_encoder_checkpoint: Optional[str] = None,
                     keep_metadata: bool = False) -> Iterator[dict]:
    """Yields ``{"image_input_ids": LongTensor[L], "encoder_hidden_states": Tensor[S, E]}`` per sample, the dict
    training/data.py:561-573 produces (extensions matched lower-cased with '/' -> '.', other members dropped)."""
    vae_key = vae_checkpoint.lower().replace("/", ".") + ".pth"
    text_key = None if text_encoder_checkpoint is None else text_encoder_checkpoint.lower().replace("/", ".") + ".pth"
    tar = tarfile.open(src, "r") if isinstance(src, str) else tarfile.open(fileobj=src, mode="r|")
    current, sample = None, {}

    def finish(s):
        if "image_input_ids" in s and (text_key is None or "encoder_hidden_states" in s):
            return s
        return None  # incomplete samples are skipped (webdataset's warn_and_continue)

    with tar:
        for member in tar:
            if not member.isreg():
                continue
            m = _SPLIT.match(member.name)
            if m is None:
                continue
            key, ext = m.group(1), m.group(2).lower()
            if key != current:
                done = finish(sample) if current is not None else None
                if done is not None:
                    yield done
                current, sample = key, {"__key__": key}
            data = tar.extractfile(member).read()
            if ext == vae_key:
                sample["image_input_ids"] = torch.load(io.BytesIO(data), weights_only=True)
            elif text_key is not None and ext == text_key:
                sample["encoder_hidden_states"] = torch.load(io.BytesIO(data), weights_only=True)
            elif keep_metadata and ext == "json":
                sample["json"] = json.loads(data.decode("utf-8"))
        done = finish(sample) if current is not None else None
        if done is not None:
            yield done


def collate_pre_encoded(samples: Iterable[dict]) -> dict:
    """default_collate of the two tensor fields (what the reference's dataloader hands to train_muse.py:689-690)."""
    samples = list(samples)
    out = {"image_input_ids": torch.stack([s["image_input_ids"] for s in samples])}
    if "encoder_hidden_states" in samples[0]:
        out["encoder_hidden_states"] = torch.stack([s["encoder_hidden_states"] for s in samples])
    return out


@torch.no_grad()
def pre_encode_images(vq_model, batches: Iterable, writer: PreEncodedShardWriter, soft_targets: bool = False) -> int:
    """Tokenise-and-write loop: ``batches`` yields ``(keys, pixel_values[B,3,R,R] in [0,1], encoder_hidden_states[B,S,E] or
    None, metadata list or None)``.  Token ids come from ``vq_model.get_code`` on the GPU; the device->host copy of batch i
    (pinned, asynchronous) overlaps the encode of batch i+1 and the tar write happens once its copy event completed --
    the reference instead parks a thread pool behind ``.to('cpu')`` (scripts/pre_encode.py:92-110)."""
    dev = next(vq_model.parameters()).device
    pending = None
    n = 0

    def flush(p):
        nonlocal n
        keys, ids_host, ehs, metas, ev = p
        ev.synchronize()
        for i, k in enumerate(keys):
            writer.write(k, ids_host[i], None if ehs is None else ehs[i], None if metas is None else metas[i])
            n += 1

    for keys, pixels, ehs, metas in batches:
        ids = vq_model.get_code(pixels.to(dev, non_blocking=True))
        host = torch.empty(ids.shape, dtype=ids.dtype, pin_memory=dev.type == "cuda")
        host.copy_(ids, non_blocking=True)
        ev = torch.cuda.Event() if dev.type == "cuda" else None
        if ev is not None:
            ev.record()
        if pending is not None:
            flush(pending)
        pending = (keys, host, ehs, metas, ev if ev is not None else _NoEvent())
    if pending is not None:
        flush(pending)
    return n


class _NoEvent:
    def synchronize(self):
        pass
