"""CPU oracle for the mean-teacher and entropy-minimisation step bodies (TEST INFRASTRUCTURE ONLY, like wsl_oracle.py).

Loss compositions of train_mean_teacher_2D.py and train_entropy_minimization_2D.py (paths relative to the reference's ``code/``),
built from wsl_oracle's restatements of DiceLoss, entropy_loss and softmax_mse_loss.  Pinned against the unmodified reference by
oracle/make_golden_semi.py and tests/golden/semi_steps.npz (tests/test_semi_steps_cpu.py)."""
import torch
import torch.nn.functional as F

from wsl_oracle import dice_loss, entropy_loss, sigmoid_rampup, softmax_mse


def supervised_half(out_l, label_l):
    """0.5 * (DiceLoss(softmax) + CrossEntropyLoss()) on the labelled batch (dense labels, no ignore_index), the supervised half
    of train_mean_teacher_2D.py:161-163 and train_entropy_minimization_2D.py:136-138"""
    loss_ce = F.cross_entropy(out_l, label_l.long())
    loss_dice = dice_loss(torch.softmax(out_l, 1), label_l.long().unsqueeze(1))
    return 0.5 * (loss_dice + loss_ce)


def mt_losses(out_l, out_u, ema_out, label_l, iter_num, consistency=0.1, consistency_rampup=200.0):
    """Loss composition of train_mean_teacher_2D.py:151-171 (-> loss, supervised, consistency, weight).
    out_l / out_u: student logits on the labelled / unlabelled batch (two forwards, :151-155); ema_out: the teacher's logits on
    the noisy unlabelled batch (:147-149, :157-159).  Runs in the dtype of its inputs (fp32 or fp64)."""
    supervised = supervised_half(out_l, label_l)                                              # :161-163
    cw = consistency * sigmoid_rampup(iter_num // 300, consistency_rampup)                    # :73-75, :164-165
    cons = softmax_mse(out_u, ema_out).mean()                                                 # :169-170
    return supervised + cw * cons, supervised, cons, cw                                       # :171


def em_losses(out_l, out_u, label_l, iter_num, consistency=0.1, consistency_rampup=200.0):
    """Loss composition of train_entropy_minimization_2D.py:130-142 (-> loss, supervised, entropy term, weight): the supervised
    half of `mt_losses` + w * losses.entropy_loss(softmax(out_u), C=4) (:141).  Runs in the dtype of its inputs."""
    supervised = supervised_half(out_l, label_l)                                              # :136-138
    cw = consistency * sigmoid_rampup(iter_num // 300, consistency_rampup)                    # :140
    ent = entropy_loss(torch.softmax(out_u, 1), C=4)                                          # :133-134, :141
    return supervised + cw * ent, supervised, ent, cw                                         # :142
