"""CPU restatement of the feature-cache (DeepCache) cheap forward, built from the oracle's blocks.

A cheap forward at level L recomputes the conditioning, the input conv, the down and up blocks of the levels below L and
the head, and reads `deep`, the output of the up ResnetBlock that leaves level L, from an earlier full forward.  The block
names follow the oracle's creation order (XUNetBlock_k, ResnetBlock_k), so `kept_blocks` says which parameters it reads."""
import torch

from oracle import xunet_ref as R


def _names(cfg: R.RefConfig):
    """Block names by role: down[i] (xblocks of down-level i), down_rs[i] (the ResnetBlock from level i to i + 1), middle,
    up[i] (xblocks of up-level i) and up_rs[i] (the ResnetBlock from level i to i - 1)."""
    n, nrb = len(cfg.ch_mult), cfg.num_res_blocks
    down = [[f'XUNetBlock_{i * nrb + k}' for k in range(nrb)] for i in range(n)]
    down_rs = [f'ResnetBlock_{i}' for i in range(n - 1)]
    middle = f'XUNetBlock_{n * nrb}'
    up = [[f'XUNetBlock_{n * nrb + 1 + (n - 1 - i) * (nrb + 1) + k}' for k in range(nrb + 1)] for i in range(n)]
    up_rs = [None] + [f'ResnetBlock_{n - 1 + n - 1 - i}' for i in range(1, n)]
    return down, down_rs, middle, up, up_rs


def cached_name(cfg: R.RefConfig, level: int) -> str:
    """The oracle tap (and engine tap) of the tensor a cheap forward at `level` reads."""
    check_level(cfg, level)
    return _names(cfg)[4][level]


def check_level(cfg: R.RefConfig, level: int) -> None:
    if not 1 <= level <= len(cfg.ch_mult) - 1:
        raise ValueError(f'level {level} outside [1, {len(cfg.ch_mult) - 1}]')


def kept_blocks(cfg: R.RefConfig, level: int) -> set:
    """Top-level parameter groups a cheap forward reads: every ConditioningProcessor_0 leaf but the pose-embedding convs of
    levels >= `level` (named 'ConditioningProcessor_0/<leaf>'), the input conv, the blocks of the levels below `level`
    (without the down ResnetBlock into `level`) and the head."""
    check_level(cfg, level)
    down, down_rs, _, up, up_rs = _names(cfg)
    keep = {'Conv_0', 'Conv_1', 'GroupNorm_0', 'ConditioningProcessor_0/Dense_0', 'ConditioningProcessor_0/Dense_1',
            'ConditioningProcessor_0/pos_emb', 'ConditioningProcessor_0/ref_pose_emb_first',
            'ConditioningProcessor_0/ref_pose_emb_other'}
    keep |= {f'ConditioningProcessor_0/Conv_{i}' for i in range(level)}
    for i in range(level):
        keep |= set(down[i]) | set(up[i])
        if i + 1 < level:
            keep.add(down_rs[i])
        if i >= 1:
            keep.add(up_rs[i])
    return keep


def shallow_forward(params, batch, cond_mask, cfg: R.RefConfig, level: int, deep, *, emu=None):
    """eps_hat (B, H, W, 3) of a cheap forward at `level`; deep: (B, 2, H', W', C') the cached tensor (`cached_name`), as an
    oracle tap.  train=False."""
    check_level(cfg, level)
    emu = emu or R._EXACT
    down, down_rs, _, up, up_rs = _names(cfg)
    dtype = batch['x'].dtype
    cp = params['ConditioningProcessor_0']
    # the deep pose-embedding convs are not evaluated: only Conv_0 .. Conv_{level-1} of the conditioning are passed on
    sub = {k: v for k, v in cp.items() if not (k.startswith('Conv_') and int(k[5:]) >= level)}
    shallow_cfg = R.RefConfig(**{**cfg.__dict__, 'ch_mult': cfg.ch_mult[:level]})
    logsnr_emb, pose_embs = R.conditioning(sub, batch, cond_mask, shallow_cfg, emu=emu)
    lemb = logsnr_emb[:, None, None, None, :]

    def xblock(name, h, i):
        return R.xunet_block(h, lemb + pose_embs[i], params[name], features=cfg.ch * cfg.ch_mult[i],
                             use_attn=h.shape[2] in cfg.attn_resolutions, heads=cfg.attn_heads, dropout=cfg.dropout,
                             train=False, drop_mask=None, emu=emu)

    def rblock(name, h, i, resample):
        return R.resnet_block(h, lemb + pose_embs[i], params[name], resample=resample, dropout=cfg.dropout, train=False,
                              drop_mask=None, emu=emu)

    h = emu.store(torch.stack([batch['x'].to(dtype), batch['z'].to(dtype)], dim=1))
    h = emu.store(R.conv_1x3x3(h, params['Conv_0']['kernel'], params['Conv_0']['bias']))
    hs = [h]
    for i in range(level):
        for name in down[i]:
            h = xblock(name, h, i)
            hs.append(h)
        if i + 1 < level:
            h = rblock(down_rs[i], h, i + 1, 'down')
            hs.append(h)
    h = deep.to(dtype)
    for i in reversed(range(level)):
        for name in up[i]:
            h = xblock(name, torch.cat([h, hs.pop()], dim=-1), i)
        if i != 0:
            h = rblock(up_rs[i], h, i - 1, 'up')
    assert not hs
    h = emu.store(R.swish(R.group_norm(h, params['GroupNorm_0'])))
    out = emu.store(R.conv_1x3x3(h, params['Conv_1']['kernel'], params['Conv_1']['bias']))
    return out[:, 1]
