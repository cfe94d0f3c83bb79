/* ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement (fp64 arithmetic, exact integers) of the arithmetic core of the reference's
 * RLHF loss path, independent of PyTorch.  Used by tests/ to cross-check oracle/ref_port.py (which
 * is pinned bit-exactly on the reference's golden vectors) and, through it, the CUDA kernels.
 * Only tests/, __graft_entry__ and bench.py's CPU legs may load this; the product never does.
 * Paths below are relative to the reference's align_anything/ directory.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* utils/tools.py:402-413: log_softmax over V then gather at the label; one value per row. */
void oracle_token_log_probs(const float *logits, const int64_t *labels, int64_t rows, int64_t V, double *out) {
  for (int64_t r = 0; r < rows; ++r) {
    const float *x = logits + r * V;
    double mx = -INFINITY;
    for (int64_t j = 0; j < V; ++j)
      if ((double)x[j] > mx) mx = (double)x[j];
    double s = 0.0;
    for (int64_t j = 0; j < V; ++j) s += exp((double)x[j] - mx);
    out[r] = ((double)x[labels[r]] - mx) - log(s);
  }
}

/* autograd of the above for upstream per-row gradient g: grad[j] = g * ([j == y] - softmax_j). */
void oracle_token_log_probs_grad(const float *logits, const int64_t *labels, const double *g, int64_t rows,
                                 int64_t V, double *grad) {
  for (int64_t r = 0; r < rows; ++r) {
    const float *x = logits + r * V;
    double mx = -INFINITY, s = 0.0;
    for (int64_t j = 0; j < V; ++j)
      if ((double)x[j] > mx) mx = (double)x[j];
    for (int64_t j = 0; j < V; ++j) s += exp((double)x[j] - mx);
    for (int64_t j = 0; j < V; ++j)
      grad[r * V + j] = g[r] * ((j == labels[r] ? 1.0 : 0.0) - exp((double)x[j] - mx) / s);
  }
}

/* trainers/text_to_text/dpo.py:172-194 for one pair given the four sequence log-prob sums. */
void oracle_dpo_pair(double pc, double pr, double rc, double rr, double beta, double *loss, double *better,
                     double *worse) {
  const double z = beta * ((pc - rc) - (pr - rr));
  *loss = -(fmin(z, 0.0) - log1p(exp(-fabs(z)))); /* -logsigmoid(z) */
  *better = beta * (pc - rc);
  *worse = beta * (pr - rr);
}

/* trainers/text_to_text/ppo.py:528-547 for one row (mask: 0/1 bytes). Returns end index or -1. */
int64_t oracle_kl_rewards(const double *lp, const double *ref, const uint8_t *mask, int64_t W, double reward,
                          double kl_coeff, double clip, double *out) {
  int64_t end = -1;
  for (int64_t t = 0; t < W; ++t)
    if (mask[t]) end = t;
  for (int64_t t = 0; t < W; ++t) {
    double r = -kl_coeff * (lp[t] - ref[t]);
    if (t == end) r += reward;
    out[t] = r > clip ? clip : (r < -clip ? -clip : r);
  }
  return end;
}

/* trainers/text_to_text/ppo.py:487-508 for one row: sequential reverse recurrence. */
void oracle_gae(const double *values, const double *rewards, const uint8_t *mask, int64_t W, int64_t start,
                double gamma, double lam, double *adv, double *ret) {
  double carry = 0.0;
  for (int64_t t = W - 1; t >= start; --t) {
    const double v = mask[t] ? values[t] : 0.0;
    const double nv = (t < W - 1 && mask[t + 1]) ? values[t + 1] : 0.0;
    const double r = mask[t] ? rewards[t] : 0.0;
    const double delta = r + gamma * nv - v;
    carry = delta + gamma * lam * carry;
    adv[t - start] = carry;
    ret[t - start] = carry + v;
  }
}

/* trainers/text_image_to_text/ppo.py:56-87: rotate each row right by the number of non-leading pads. */
void oracle_move_padding_left(const int64_t *ids, int64_t B, int64_t L, int64_t pad, int64_t *out) {
  for (int64_t b = 0; b < B; ++b) {
    const int64_t *row = ids + b * L;
    int64_t kept = 0, leading = 0;
    int seen = 0;
    for (int64_t c = 0; c < L; ++c) {
      if (row[c] != pad) {
        ++kept;
        seen = 1;
      } else if (!seen) {
        ++leading;
      }
    }
    const int64_t shift = L - kept - leading;
    for (int64_t c = 0; c < L; ++c) {
      int64_t src = (c - shift) % L;
      if (src < 0) src += L;
      out[b * L + c] = row[src];
    }
  }
}

/* trainers/text_to_text/dpo.py:52-54,135-137: the last R tokens != pad.  Returns how many were found. */
int64_t oracle_strip_pad_tail(const int64_t *row, int64_t L, int64_t pad, int64_t R, int64_t *out) {
  int64_t found = 0;
  for (int64_t c = L - 1; c >= 0 && found < R; --c)
    if (row[c] != pad) out[R - 1 - found++] = row[c];
  return found;
}

/* ---- sibling losses (SURVEY.md 8f row 2), one pair / one token each, fp64 ---------------------------------- */
static double neg_logsigmoid(double z) { return -(fmin(z, 0.0) - log1p(exp(-fabs(z)))); }

/* trainers/text_to_text/simpo.py:78-92: length-normalised log-ratios, margin gamma. */
void oracle_simpo_pair(double better_sum, double worse_sum, double better_len, double worse_len, double beta,
                       double gamma, double *loss, double *better, double *worse) {
  const double b = better_sum / better_len, w = worse_sum / worse_len;
  *loss = neg_logsigmoid(beta * (b - w) - gamma);
  *better = beta * b;
  *worse = beta * w;
}

/* trainers/text_to_text/orpo.py:78-97: SFT term + beta * odds-ratio term. */
void oracle_orpo_pair(double better_sum, double worse_sum, double better_len, double worse_len, double beta,
                      double *loss, double *better, double *worse) {
  const double b = better_sum / better_len, w = worse_sum / worse_len;
  const double log_odds = (b - w) - (log1p(-exp(b)) - log1p(-exp(w)));
  *loss = -b + beta * neg_logsigmoid(log_odds);
  *better = beta * b;
  *worse = beta * w;
}

/* trainers/text_to_text/kto.py:119-137. */
void oracle_kto_pair(double better, double ref_better, double worse, double ref_worse, double beta,
                     double scale_better, double scale_worse, double kl, double *loss, double *r_better,
                     double *r_worse) {
  const double b = better - ref_better, w = worse - ref_worse;
  *loss = scale_better * (1.0 - 1.0 / (1.0 + exp(-beta * (b - kl)))) -
          scale_worse * (1.0 - 1.0 / (1.0 + exp(-beta * (kl - w))));
  *r_better = beta * b;
  *r_worse = beta * w;
}

/* trainers/text_to_text/rm.py:112-126: -logsigmoid(higher - lower) [+ regularisation * (h^2 + l^2) in the
 * reference's mean form is applied by the caller]. */
double oracle_rm_pair(double higher_end, double lower_end) { return neg_logsigmoid(higher_end - lower_end); }

/* trainers/text_to_text/grpo.py:290-297 for one token: k3 KL and the per-token loss (exp(lp - lp.detach()) == 1). */
void oracle_grpo_token(double lp, double ref_lp, double advantage, double beta, double *kl, double *loss,
                       double *dloss_dlp) {
  const double d = ref_lp - lp;
  *kl = exp(d) - d - 1.0;
  *loss = -(advantage - beta * (*kl));
  *dloss_dlp = -(advantage) + beta * (1.0 - exp(d)); /* d/dlp of -(e^{lp - sg(lp)} A - beta kl) */
}

/* trainers/text_to_text/grpo.py:268-274: (r - group mean) / (unbiased group std + 1e-4). */
void oracle_group_advantages(const double *rewards, int64_t n_groups, int64_t group, double *adv) {
  for (int64_t g = 0; g < n_groups; ++g) {
    double mean = 0.0, var = 0.0;
    for (int64_t i = 0; i < group; ++i) mean += rewards[g * group + i];
    mean /= (double)group;
    for (int64_t i = 0; i < group; ++i) {
      const double d = rewards[g * group + i] - mean;
      var += d * d;
    }
    const double sd = sqrt(var / (double)(group - 1));
    for (int64_t i = 0; i < group; ++i) adv[g * group + i] = (rewards[g * group + i] - mean) / (sd + 1e-4);
  }
}

/* trainers/text_image_to_text/saferlhf.py:432-451: Lagrangian advantage mix and the clipped surrogate of one token. */
double oracle_saferlhf_actor_token(double lp, double old_lp, double reward_adv, double cost_adv, double multiplier,
                                   double clip) {
  const double adv = (reward_adv - multiplier * cost_adv) / (1.0 + multiplier);
  const double ratio = exp(lp - old_lp);
  const double clipped = ratio < 1.0 - clip ? 1.0 - clip : (ratio > 1.0 + clip ? 1.0 + clip : ratio);
  return -fmin(adv * ratio, adv * clipped);
}
