"""TEST INFRASTRUCTURE - plain-torch restatement of the reference's optimal-transport distance (mmf/modules/ot.py), the
checker of the word-region-alignment kernels (mmf_b200/csrc/ot.cu).  Like oracle/fusion_oracle.py it is not part of the
product: tests and tools/bench_uniter.py (as the timed torch arm) import it, mmf_b200/ never does.  It is pinned against
the reference's own cost_matrix_cosine / ipot / trace by tests/golden/uniter_model.pt (tests/test_uniter_model_cpu.py)."""
import torch
import torch.nn.functional as F


def optimal_transport_dist(txt_emb, img_emb, txt_pad, img_pad, beta=0.5, iteration=50, k=1, return_all=False):
    """optimal_transport_dist, mmf/modules/ot.py:80-102, in the dtype of its inputs (fp64 for the checker):
    cost_matrix_cosine (:15-25), the padded-pair masking (:92-93), ipot (:37-77, on the detached cost) and
    trace(cost @ T) (:28-34, 101).  txt_emb [B, M, D], img_emb [B, N, D]; txt_pad [B, M], img_pad [B, N] bool, True on
    padding.  Returns distance [B], or (distance, cost [B, M, N], T [B, N, M]) with return_all.
    k > 1: the reference's second inner pass multiplies Q by the row vector sigma it has just made and raises a shape
    error unless M = 1 (:72-74); here sigma is viewed as a column in every inner pass, the evident intent, which is the
    reference's arithmetic wherever the reference runs."""
    x_norm = F.normalize(txt_emb, p=2, dim=-1, eps=1e-5)                                   # :21-24
    y_norm = F.normalize(img_emb, p=2, dim=-1, eps=1e-5)
    cost = 1 - x_norm.matmul(y_norm.transpose(1, 2))
    joint_pad = txt_pad.unsqueeze(-1) | img_pad.unsqueeze(-2)                              # :92-96
    cost = cost.masked_fill(joint_pad, 0)
    x_len = (txt_pad.size(1) - txt_pad.sum(dim=1)).to(cost.dtype)
    y_len = (img_pad.size(1) - img_pad.sum(dim=1)).to(cost.dtype)
    with torch.no_grad():                                                                  # ipot, :50-77
        C = cost.detach()
        b, m, n = C.size()
        sigma = torch.ones(b, m, dtype=C.dtype, device=C.device) / x_len.unsqueeze(1)
        T = torch.ones(b, n, m, dtype=C.dtype, device=C.device)
        A = torch.exp(-C.transpose(1, 2) / beta)
        sigma = sigma.masked_fill(txt_pad, 0)
        jp = joint_pad.transpose(1, 2)
        T = T.masked_fill(jp, 0)
        A = A.masked_fill(jp, 0)
        xl, yl = x_len.view(b, 1, 1), y_len.view(b, 1, 1)
        x_mask = (txt_pad.to(C.dtype) * 1e4).unsqueeze(1)
        y_mask = (img_pad.to(C.dtype) * 1e4).unsqueeze(1)
        for _ in range(iteration):
            Q = A * T
            for _ in range(k):
                delta = 1 / (yl * Q.matmul(sigma.view(b, m, 1)).view(b, 1, n) + y_mask)
                sigma = 1 / (xl * delta.matmul(Q) + x_mask)
            T = delta.view(b, n, 1) * Q * sigma
        T = T.masked_fill(jp, 0)
    distance = torch.diagonal(cost.matmul(T), dim1=-2, dim2=-1).sum(-1)                    # trace, :28-34, 101
    return (distance, cost, T) if return_all else distance
