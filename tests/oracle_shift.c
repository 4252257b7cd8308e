/*
 * oracle_shift.c — the context shift on the CPU oracle's side (test infrastructure, like the oracle itself).
 *
 * oc_seq_shift restates cl_seq_shift's contract on an oracle sequence.  The oracle's sequence and model structs are private
 * to llama_oracle.c, so this file compiles that source into the same shared object: the functions below use its own struct
 * definitions and its own cos/sin table, with no second copy of either layout.  tests/shift_util.py builds it with the
 * oracle Makefile's flags plus -ffp-contract=off (the rotation's products and sums are rounded one by one, as in
 * kv_shift_kernel) and -fvisibility=hidden, so that only the two functions below are exported, and calls them on the
 * handles oracle/oracle.py hands out.
 */
#include "../oracle/llama_oracle.c"

#define OC_SHIFT_API __attribute__((visibility("default")))

/* Tokens [n_keep, n_keep + n_discard) leave the sequence: position p >= n_keep takes what p + n_discard held, V unchanged,
 * K = bf16(R(-n_discard) K_old) in fp32 (a c + b s, b c - a s for the pair of dims j, j + hd/2) with row n_discard of the
 * model's table; len drops by n_discard.  Returns 0, or -1 for arguments cl_seq_shift refuses (n_discard need not be a
 * multiple of a page here: the oracle has no pages). */
OC_SHIFT_API int oc_seq_shift(oc_seq* s, int32_t n_keep, int32_t n_discard) {
  const oc_config* c = &s->m->c;
  if (n_keep < 0 || n_discard <= 0 || n_keep + n_discard > s->len || n_discard >= c->max_seq_len) return -1;
  const int half = c->head_dim / 2, kvd = c->n_kv_heads * c->head_dim;
  const float* tab = s->m->rope + (size_t)n_discard * half * 2;
  for (int l = 0; l < c->n_layers; ++l) {
    float* kb = s->kc + (size_t)l * s->max_len * kvd;
    float* vb = s->vc + (size_t)l * s->max_len * kvd;
    for (int p = n_keep; p + n_discard < s->len; ++p) {
      const float* ks = kb + (size_t)(p + n_discard) * kvd;
      float* kd = kb + (size_t)p * kvd;
      for (int g = 0; g < c->n_kv_heads; ++g)
        for (int i = 0; i < half; ++i) {
          const float a = ks[g * c->head_dim + i], b = ks[g * c->head_dim + i + half];
          const float cs = tab[2 * i], sn = tab[2 * i + 1];
          const float ac = a * cs, bs = b * sn, bc = b * cs, as = a * sn;
          kd[g * c->head_dim + i] = oc_bf16_round(ac + bs);
          kd[g * c->head_dim + i + half] = oc_bf16_round(bc - as);
        }
      memcpy(vb + (size_t)p * kvd, vb + (size_t)(p + n_discard) * kvd, (size_t)kvd * 4);
    }
  }
  s->len -= n_discard;
  return 0;
}

/* Row `row` of the model's cos/sin table: out[head_dim / 2][2].  Returns 0, or -1 for a row outside the table. */
OC_SHIFT_API int oc_rope_row(const oc_model* m, int32_t row, float* out) {
  if (row < 0 || row >= m->c.max_seq_len) return -1;
  memcpy(out, m->rope + (size_t)row * m->c.head_dim, (size_t)m->c.head_dim * 4);
  return 0;
}
