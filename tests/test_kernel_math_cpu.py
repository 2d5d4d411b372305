"""CPU: the algebra behind four kernels, restated in numpy / torch exactly as the CUDA code computes it and checked against
the reference-side formulation (the kernels themselves are checked on the GPU; these tests keep the derivations honest in the
no-GPU suite):

 * prompt_feat.cu: kaldi fbank with DC removal + pre-emphasis + povey window + zero-padded DFT folded into ONE constant matrix applied to
   three rows of 160 samples; whisper framing as three rows of the reflect-padded signal;
 * attention_tc.cu (relpos_u_kernel + BIAS): the conformer's rel_shift as the index map U[i][center - i + j];
 * attention_tc.cu (attn_wg_kernel): the register-resident online softmax - the four lanes of a quad own interleaved key columns,
   share one running maximum per row through quad shuffles, keep partial row sums merged at the end - == softmax(S) V;
 * flow.cu (streaming sessions): a causal convolution over [saved two-row tail | chunk] == the chunk's rows of the convolution over the
   whole sequence."""
import math

import numpy as np
import torch

from oracle import flow as oflow, prompt_feat as opf


def _kaldi_matrix():
    """prompt_feat.cu::build, kaldi part: rows k2 < 257 cos, else -sin; M = DFT512 . diag(povey) . pre-emphasis . (I - 11^T/400)"""
    WIN, NFFT, NB = 400, 512, 257
    n = np.arange(WIN)
    win = (0.5 - 0.5 * np.cos(2 * np.pi * n / (WIN - 1))) ** 0.85
    M = np.zeros((2 * NB, 480))
    for k2 in range(2 * NB):
        k = k2 if k2 < NB else k2 - NB
        ang = 2 * np.pi * ((k * n) % NFFT) / NFFT
        r = np.append(win * (np.cos(ang) if k2 < NB else -np.sin(ang)), 0.0)
        q = r[:WIN] - 0.97 * r[1:WIN + 1]
        q[0] -= 0.97 * r[0]
        M[k2, :WIN] = q - q.mean()
    return M.astype(np.float32)


def test_kaldi_fbank_as_one_folded_matrix(golden):
    g = golden("prompt_feat")
    M = _kaldi_matrix()
    banks = np.pad(opf._kaldi_mel_banks(), ((0, 0), (0, 1))).astype(np.float32)
    for i in (0, 1):
        w = g[f"wave{i}"].astype(np.float32)
        m = 1 + (w.size - 400) // 160
        rows = np.zeros((m + 2) * 160, dtype=np.float32)
        rows[:min(rows.size, w.size)] = w[:rows.size]
        rows = rows.reshape(m + 2, 160)
        frames = np.concatenate([rows[:-2], rows[1:-1], rows[2:]], 1)          # frame t = rows t, t+1, t+2 (480 samples, last 80 unused)
        spec = frames @ M.T
        power = spec[:, :257] ** 2 + spec[:, 257:] ** 2
        feat = np.log(np.maximum(power @ banks.T, np.finfo(np.float32).eps))
        feat = feat - feat.mean(0, keepdims=True)
        assert feat.shape == g[f"kaldi{i}"].shape
        assert np.abs(feat - g[f"kaldi{i}"]).max() < 5e-3


def test_whisper_framing_as_three_rows_of_the_reflect_padded_signal(golden):
    g = golden("prompt_feat")
    w = torch.from_numpy(g["wave1"])
    T = w.numel() // 160
    idx = torch.arange((T + 2) * 160) - 200                                    # rows160_kernel with pad 200
    idx = idx.abs()
    idx = torch.where(idx >= w.numel(), 2 * (w.numel() - 1) - idx, idx)
    rows = w[idx].view(T + 2, 160)
    frames = torch.cat([rows[:-2], rows[1:-1], rows[2:]], 1)[:, :400]
    win = torch.hann_window(400)
    mag = torch.fft.rfft(frames * win).abs() ** 2                              # [T, 201]
    ref = torch.stft(w, 400, 160, window=win, return_complex=True)[..., :-1].abs() ** 2
    assert mag.shape == ref.t().shape
    assert (mag - ref.t()).abs().max() < 1e-3 * ref.abs().max()


def test_rel_shift_is_the_index_map_center_minus_i_plus_j():
    g = torch.Generator().manual_seed(0)
    T, H, d = 37, 2, 8
    qv = torch.randn(1, H, T, d, generator=g)
    pp = torch.randn(1, H, 2 * T - 1, d, generator=g)                          # rows m = 0..2T-2 hold relative position T-1-m
    bd = oflow._rel_shift(torch.matmul(qv, pp.transpose(-2, -1)))              # reference: [1,H,T,T]
    U = torch.matmul(qv, pp.transpose(-2, -1))                                 # relpos_u_kernel: un-shifted [T, 2T-1]
    center = T - 1
    i = torch.arange(T)[:, None]
    j = torch.arange(T)[None, :]
    bias = U[0][:, i, center - i + j]                                          # attn_wg_kernel<BIAS>: ubias[.. + center - i + j]
    assert torch.equal(bias, bd[0])


def test_quad_online_softmax_equals_softmax():
    """attn_wg_kernel: per 64-key tile, quad lane q holds the scores of keys 8 jj + 2 q + e (jj < 8, e < 2) of its row; the row maximum
    is the quad maximum of the lane maxima (log2 units), the accumulator and the per-lane sums are rescaled by 2^(m_old - m_new) when
    the maximum grows, keys past the row's limit are -inf (P = 0), and the row sum is the quad sum of the lane sums at the end"""
    g = torch.Generator().manual_seed(1)
    d, scale = 16, 0.125 * math.log2(math.e)
    rescales = 0
    for trial, (L, klim) in enumerate(((300, 300), (300, 250), (64, 1), (130, 100))):
        s = torch.randn(L, generator=g, dtype=torch.float64) * 3.0 + torch.arange(L, dtype=torch.float64) * (0.5 * trial)   # a rising trend forces rescales
        V = torch.randn(L, d, generator=g, dtype=torch.float64)
        ref = torch.softmax(s[:klim] * 0.125, 0) @ V[:klim]
        m = -math.inf
        lane_sum = [0.0] * 4
        O = torch.zeros(d, dtype=torch.float64)
        for j0 in range(0, L, 64):
            cols = [[j0 + 8 * jj + 2 * q + e for jj in range(8) for e in range(2)] for q in range(4)]
            x = [[(s[j].item() if j < klim else -math.inf) for j in cols[q] if j < L] for q in range(4)]
            mt = max(max(xs, default=-math.inf) for xs in x) * scale                  # quad_max of the lane maxima
            mn = max(m, mt)
            f = 1.0 if m == -math.inf else 2.0 ** (m - mn)
            if f != 1.0:
                rescales += 1
            m = mn
            mneg = 0.0 if mn == -math.inf else -mn
            O *= f
            for q in range(4):
                lane_sum[q] *= f
                for j, xv in zip(cols[q], x[q]):
                    p = 0.0 if xv == -math.inf else 2.0 ** (xv * scale + mneg)
                    lane_sum[q] += p
                    O += p * V[j]
        den = sum(lane_sum)                                                             # quad_sum at the end
        out = O / den
        assert (out - ref).abs().max() < 1e-12
    assert rescales > 0


def test_causal_conv_over_saved_tail_plus_chunk_equals_the_whole_sequence():
    """conv_state_kernel: the two rows a causal k=3 convolution reads in front of a chunk are the last two INPUT rows of the previous chunk
    (zeros before the first); k=31 (DiT position convolution): thirty rows"""
    g = torch.Generator().manual_seed(2)
    for k in (3, 31):
        C, T = 5, 150
        x = torch.randn(1, C, T, generator=g, dtype=torch.float64)
        w = torch.randn(4, C, k, generator=g, dtype=torch.float64)
        ref = torch.nn.functional.conv1d(torch.nn.functional.pad(x, (k - 1, 0)), w)
        tail = torch.zeros(1, C, k - 1, dtype=torch.float64)
        outs = []
        for a, b in ((0, 50), (50, 100), (100, 150)):
            chunk = x[:, :, a:b]
            outs.append(torch.nn.functional.conv1d(torch.cat([tail, chunk], 2), w))
            tail = chunk[:, :, -(k - 1):]
        assert torch.equal(torch.cat(outs, 2), ref)
