"""Golden fixtures larger than PART_BYTES are stored as <stem>.pt plus <stem>.part<i>.pt: every file stays small enough
for the repository, the content is unchanged.  load_golden() reassembles the dict that save_golden() was given.

Large activations are stored at a sample of pixel positions (stage_positions, sample_stage) and full-size maps in bands
of rows (bands, unband): the part splitter moves whole entries, so each band is an entry of its own."""
import glob
import io
import os

import numpy as np
import torch

from oracle import synth

PART_BYTES = 900 * 1024


def _nbytes(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    return len(buf.getvalue())


def save_golden(g, path):
    """torch.save(g, path), moving entries (or entries of dict-valued entries) into part files while path is too big."""
    stem = path[:-3]
    for old in glob.glob(glob.escape(stem) + ".part*.pt"):
        os.remove(old)
    items = []  # (top key, sub key or None, value)
    for k, v in g.items():
        if isinstance(v, dict) and _nbytes(v) > PART_BYTES // 4:
            items += [(k, sk, sv) for sk, sv in v.items()]
        else:
            items.append((k, None, v))
    parts, cur, cur_bytes = [], [], 0
    for it in items:
        n = _nbytes(it[2])
        if cur and cur_bytes + n > PART_BYTES:
            parts.append(cur)
            cur, cur_bytes = [], 0
        cur.append(it)
        cur_bytes += n
    parts.append(cur)

    def pack(its):
        out = {}
        for k, sk, v in its:
            if sk is None:
                out[k] = v
            else:
                out.setdefault(k, {})[sk] = v
        return out

    torch.save(pack(parts[0]), path)
    for i, its in enumerate(parts[1:], 1):
        torch.save(pack(its), f"{stem}.part{i}.pt")


def stage_positions(prefix, seed, floats, h, w, channels):
    """sorted flat pixel indices (row-major over h x w) at which a stage of `channels` channels is stored: about
    `floats` values, at least one position"""
    n = min(h * w, max(1, floats // channels))
    rs = synth._rs(f"{prefix}.positions.{h}x{w}x{channels}", seed)
    return np.sort(rs.choice(h * w, n, replace=False))


def sample_stage(t, idx):
    """fp32 [1, C, h, w] stage -> [C, len(idx)] at the given flat pixel indices"""
    return t[0].reshape(t.shape[1], -1)[:, torch.as_tensor(idx, device=t.device)].float().cpu().contiguous()


def bands(t, rows):
    """[H, ...] -> {band name: `rows` rows}"""
    return {f"rows{r:05d}": t[r:r + rows].clone() for r in range(0, t.shape[0], rows)}


def unband(d):
    """the tensor that `bands` split"""
    return torch.cat([d[k] for k in sorted(d)])


def load_golden(path):
    g = torch.load(path, weights_only=False)
    for part in sorted(glob.glob(glob.escape(path[:-3]) + ".part*.pt")):
        for k, v in torch.load(part, weights_only=False).items():
            if isinstance(v, dict) and isinstance(g.get(k), dict):
                g[k].update(v)
            else:
                g[k] = v
    return g
