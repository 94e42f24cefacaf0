"""TEST INFRASTRUCTURE: the torch-CPU emulation of tests/emu_backend.py extended with espb_softmax_rows_split_f32, so that the intermediate-CTC
host logic of espnet_b200/layers.py (EncoderBase._interctc) runs on a box without a GPU.  Restates the contract in include/espnet_b200.h."""
import torch

import emu_backend as emu


def _softmax_rows_split(x, rows, ld, V, out, out_plane, ldo):
    assert V > 0 and ld >= V and ldo >= V and ldo % 32 == 0 and out_plane >= rows * ldo
    p = torch.zeros(rows, ldo)
    p[:, :V] = torch.softmax(torch.as_strided(x, (rows, V), (ld, 1), x.storage_offset()), dim=-1)
    emu._store(emu._flat(out), torch.arange(rows * ldo).view(rows, ldo), p, True, out_plane)


def install(monkeypatch):
    """emu_backend.install + the softmax into the split layout."""
    emu.install(monkeypatch)
    monkeypatch.setitem(emu._TABLE, "espb_softmax_rows_split_f32", _softmax_rows_split)
