/*
 * ORACLE — TEST INFRASTRUCTURE ONLY (see lyra_oracle.h).
 *
 * A small interpreter for the two streaming conv-net graphs of the reference,
 *   lyra/model_coeffs/soundstream_encoder.tflite   (reference call site: lyra/soundstream_encoder.cc:53-64)
 *   lyra/model_coeffs/lyragan.tflite               (reference call site: lyra/lyra_gan_model.cc:53-64)
 * which the reference executes with tflite::Interpreter::Invoke (lyra/tflite_model_wrapper.cc:102-104).
 * TensorFlow Lite v2.11.0 (commit d5b57ca93e506df258271ea00fc29cf98383a374, reference WORKSPACE:168-174)
 * is NOT vendored in the reference repository, so each builtin op is restated here from TFLite's published
 * *reference kernels* (tensorflow/lite/kernels/internal/reference/{conv,depthwiseconv_float,
 * transpose_conv,leaky_relu,add,sub,quantize,dequantize,concatenation,strided_slice}.h and
 * reference/integer_ops/{conv,depthwise_conv,transpose_conv,add}.h), including the gemmlowp
 * fixed-point requantisation (MultiplyByQuantizedMultiplier, double-rounding variant).
 *
 * Canonical fp32 arithmetic (the reference's XNNPACK summation order is unknowable offline,
 * SURVEY.md §0.8): every fp32 convolution output is ONE fused-multiply-add chain
 *     acc = +0;  for k ascending, for cin ascending:  acc = fmaf(x, w, acc);  out = acc + bias
 * (for TRANSPOSE_CONV: input position ascending, then cin ascending — the loop order of the TFLite
 * reference kernel).  The CUDA product reproduces exactly this chain, so GPU == oracle bit-for-bit.
 * Everything else (LeakyReLU, ADD, SUB, QUANTIZE, DEQUANTIZE) is a single correctly-rounded IEEE op.
 * Compile with -ffp-contract=off: only the explicit fmaf() calls may fuse.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "lyra_oracle.h"
#include "tfl_reader.h"

/* ---------------------------------------------------------------- fixed point (gemmlowp) ---- */

/* tensorflow/lite/kernels/internal/quantization_util.cc: QuantizeMultiplier */
void lo_quantize_multiplier(double d, int32_t* qm, int* shift) {
  if (d == 0.0) { *qm = 0; *shift = 0; return; }
  const double q = frexp(d, shift);
  int64_t q_fixed = (int64_t)round(q * (double)(1ll << 31));
  if (q_fixed == (1ll << 31)) { q_fixed /= 2; ++*shift; }
  if (*shift < -31) { *shift = 0; q_fixed = 0; }
  *qm = (int32_t)q_fixed;
}

/* gemmlowp fixedpoint.h: SaturatingRoundingDoublingHighMul */
static inline int32_t srdhm(int32_t a, int32_t b) {
  const int overflow = (a == b) && (a == INT32_MIN);
  const int64_t ab = (int64_t)a * (int64_t)b;
  const int32_t nudge = ab >= 0 ? (1 << 30) : (1 - (1 << 30));
  const int32_t r = (int32_t)((ab + nudge) / (1ll << 31));
  return overflow ? INT32_MAX : r;
}
/* gemmlowp fixedpoint.h: RoundingDivideByPOT */
static inline int32_t rdbpot(int32_t x, int exponent) {
  const int32_t mask = (int32_t)((1ll << exponent) - 1);
  const int32_t remainder = x & mask;
  const int32_t threshold = (mask >> 1) + (x < 0 ? 1 : 0);
  return (x >> exponent) + (remainder > threshold ? 1 : 0);
}
/* tensorflow/lite/kernels/internal/common.h: MultiplyByQuantizedMultiplier (no TFLITE_SINGLE_ROUNDING) */
int32_t lo_mbqm(int32_t x, int32_t qm, int shift) {
  const int left = shift > 0 ? shift : 0;
  const int right = shift > 0 ? 0 : -shift;
  return rdbpot(srdhm(x * (1 << left), qm), right);
}
static inline int32_t clamp_i8(int32_t v) { return v < -128 ? -128 : (v > 127 ? 127 : v); }

/* ---------------------------------------------------------------- runtime structures ---- */

typedef struct {
  char name[128];
  float* data;
  size_t count;
} lo_var;

typedef struct {
  /* conv-like geometry */
  int K, stride, dil, Cin, Cout, groups, CinG, CoutG, Tin, Tout;
  float* wf;        /* f32 weights, [g][k][ci][coG]  (transposed conv: [k][ci][co]) */
  int8_t* wq;       /* int8 weights, same layouts */
  const float* bf;
  const int32_t* bq;
  int32_t* qm;      /* per-output-channel multiplier / shift */
  int* qs;
  int32_t in_off, out_off;
  /* elementwise quant params */
  int32_t m1, m2, m3;
  int s1, s2, s3, left_shift;
  int32_t in2_off;
  float alpha;
  int var;          /* variable index for VAR_HANDLE / READ / ASSIGN */
  int32_t* scratch; /* int32 accumulators for int8 transposed conv */
} op_prep;

struct lo_net {
  tfl_model* m;
  tfl_subgraph* sg;
  void** buf;       /* per-tensor runtime storage (NULL for constants / resources) */
  int* var_of;      /* per-tensor variable index for resource tensors */
  op_prep* prep;
  lo_var vars[64];
  int nvars;
};

static int esize(int type) {
  switch (type) {
    case TFL_F32: case TFL_I32: return 4;
    case TFL_I64: return 8;
    case TFL_I8: case TFL_U8: case TFL_BOOL: return 1;
    default: return 0;
  }
}
static const void* tdata(const lo_net* n, int i) {
  const tfl_tensor* t = &n->sg->tensors[i];
  return t->data ? (const void*)t->data : (const void*)n->buf[i];
}
static void* tbuf(lo_net* n, int i) { return n->buf[i]; }

static int find_var(lo_net* n, const char* s, int len) {
  for (int i = 0; i < n->nvars; ++i)
    if ((int)strlen(n->vars[i].name) == len && memcmp(n->vars[i].name, s, (size_t)len) == 0) return i;
  return -1;
}
static int add_var(lo_net* n, const char* s, int len) {
  int v = find_var(n, s, len);
  if (v >= 0) return v;
  if (n->nvars >= 64 || len >= 127) return -1;
  v = n->nvars++;
  memcpy(n->vars[v].name, s, (size_t)len);
  n->vars[v].name[len] = 0;
  n->vars[v].data = NULL;
  n->vars[v].count = 0;
  return v;
}


/* ---------------------------------------------------------------- op preparation ---- */

static int prep_conv(lo_net* n, const tfl_op* op, op_prep* p) {
  const tfl_tensor* T = n->sg->tensors;
  const tfl_tensor *x = &T[op->in[0]], *w = &T[op->in[1]], *b = &T[op->in[2]], *y = &T[op->out[0]];
  if (x->ndim != 4 || w->ndim != 4 || w->shape[2] != 1 || x->shape[2] != 1) return -1;
  /* Conv2DOptions{0 padding, 1 stride_w, 2 stride_h, 3 act, 4 dilation_w, 5 dilation_h}; VALID only */
  p->stride = tfl_opt_i32(n->m, op, 2, 1);
  p->dil = tfl_opt_i32(n->m, op, 5, 1);
  if (tfl_opt_i8(n->m, op, 0, 0) != 1 || tfl_opt_i8(n->m, op, 3, 0) != 0) return -1;
  p->Cout = w->shape[0]; p->K = w->shape[1]; p->CinG = w->shape[3];
  p->Cin = x->shape[3];
  p->groups = p->Cin / p->CinG;            /* TFLite grouped CONV_2D: groups = input_depth / filter_input_depth */
  p->CoutG = p->Cout / p->groups;
  p->Tin = x->shape[1]; p->Tout = y->shape[1];
  if (p->Tout != (p->Tin - (p->K - 1) * p->dil - 1) / p->stride + 1) return -1;
  const size_t nw = (size_t)p->Cout * p->K * p->CinG;
  if (w->type == TFL_F32) {
    const float* src = (const float*)w->data;
    p->wf = (float*)malloc(nw * sizeof(float));
    for (int co = 0; co < p->Cout; ++co) {
      const int g = co / p->CoutG, cg = co % p->CoutG;
      for (int k = 0; k < p->K; ++k)
        for (int ci = 0; ci < p->CinG; ++ci)
          p->wf[(((size_t)g * p->K + k) * p->CinG + ci) * p->CoutG + cg] = src[((size_t)co * p->K + k) * p->CinG + ci];
    }
    p->bf = (const float*)b->data;
  } else if (w->type == TFL_I8) {
    const int8_t* src = (const int8_t*)w->data;
    p->wq = (int8_t*)malloc(nw);
    for (int co = 0; co < p->Cout; ++co) {
      const int g = co / p->CoutG, cg = co % p->CoutG;
      for (int k = 0; k < p->K; ++k)
        for (int ci = 0; ci < p->CinG; ++ci)
          p->wq[(((size_t)g * p->K + k) * p->CinG + ci) * p->CoutG + cg] = src[((size_t)co * p->K + k) * p->CinG + ci];
    }
    p->bq = (const int32_t*)b->data;
    p->qm = (int32_t*)malloc(sizeof(int32_t) * (size_t)p->Cout);
    p->qs = (int*)malloc(sizeof(int) * (size_t)p->Cout);
    /* kernel_util.cc PopulateConvolutionQuantizationParams */
    for (int co = 0; co < p->Cout; ++co) {
      const float fs = w->scale[w->nscale > 1 ? co : 0];
      const double eff = (double)x->scale[0] * (double)fs / (double)y->scale[0];
      lo_quantize_multiplier(eff, &p->qm[co], &p->qs[co]);
    }
    p->in_off = -(int32_t)x->zero_point[0];
    p->out_off = (int32_t)y->zero_point[0];
  } else {
    return -1;
  }
  return 0;
}

static int prep_dw(lo_net* n, const tfl_op* op, op_prep* p) {
  const tfl_tensor* T = n->sg->tensors;
  const tfl_tensor *x = &T[op->in[0]], *w = &T[op->in[1]], *b = &T[op->in[2]], *y = &T[op->out[0]];
  /* DepthwiseConv2DOptions{0 padding, 1 stride_w, 2 stride_h, 3 depth_multiplier, 4 act, 5 dil_w, 6 dil_h} */
  p->stride = tfl_opt_i32(n->m, op, 2, 1);
  p->dil = tfl_opt_i32(n->m, op, 6, 1);
  if (tfl_opt_i8(n->m, op, 0, 0) != 1 || tfl_opt_i32(n->m, op, 3, 1) != 1 || p->stride != 1) return -1;
  p->K = w->shape[1]; p->Cin = p->Cout = w->shape[3];
  p->Tin = x->shape[1]; p->Tout = y->shape[1];
  if (p->Tout != p->Tin - (p->K - 1) * p->dil) return -1;
  if (w->type == TFL_F32) {
    p->wf = (float*)malloc(sizeof(float) * (size_t)p->K * p->Cin);
    memcpy(p->wf, w->data, sizeof(float) * (size_t)p->K * p->Cin);
    p->bf = (const float*)b->data;
  } else {
    p->wq = (int8_t*)malloc((size_t)p->K * p->Cin);
    memcpy(p->wq, w->data, (size_t)p->K * p->Cin);
    p->bq = (const int32_t*)b->data;
    p->qm = (int32_t*)malloc(sizeof(int32_t) * (size_t)p->Cout);
    p->qs = (int*)malloc(sizeof(int) * (size_t)p->Cout);
    for (int c = 0; c < p->Cout; ++c) {
      const float fs = w->scale[w->nscale > 1 ? c : 0];
      const double eff = (double)x->scale[0] * (double)fs / (double)y->scale[0];
      lo_quantize_multiplier(eff, &p->qm[c], &p->qs[c]);
    }
    p->in_off = -(int32_t)x->zero_point[0];
    p->out_off = (int32_t)y->zero_point[0];
  }
  return 0;
}

static int prep_tconv(lo_net* n, const tfl_op* op, op_prep* p) {
  const tfl_tensor* T = n->sg->tensors;
  /* TRANSPOSE_CONV inputs: output_shape, weights [Cout,K,1,Cin], input, bias */
  const tfl_tensor *w = &T[op->in[1]], *x = &T[op->in[2]], *b = &T[op->in[3]], *y = &T[op->out[0]];
  /* TransposeConvOptions{0 padding, 1 stride_w, 2 stride_h} */
  p->stride = tfl_opt_i32(n->m, op, 2, 1);
  if (tfl_opt_i8(n->m, op, 0, 0) != 1) return -1;
  p->Cout = w->shape[0]; p->K = w->shape[1]; p->Cin = w->shape[3];
  p->Tin = x->shape[1]; p->Tout = y->shape[1];
  if (p->Tout != (p->Tin - 1) * p->stride + p->K || x->shape[3] != p->Cin) return -1;
  const size_t nw = (size_t)p->Cout * p->K * p->Cin;
  if (w->type == TFL_F32) {
    const float* src = (const float*)w->data;
    p->wf = (float*)malloc(nw * sizeof(float));
    for (int co = 0; co < p->Cout; ++co)
      for (int k = 0; k < p->K; ++k)
        for (int ci = 0; ci < p->Cin; ++ci)
          p->wf[((size_t)k * p->Cin + ci) * p->Cout + co] = src[((size_t)co * p->K + k) * p->Cin + ci];
    p->bf = (const float*)b->data;
  } else {
    const int8_t* src = (const int8_t*)w->data;
    p->wq = (int8_t*)malloc(nw);
    for (int co = 0; co < p->Cout; ++co)
      for (int k = 0; k < p->K; ++k)
        for (int ci = 0; ci < p->Cin; ++ci)
          p->wq[((size_t)k * p->Cin + ci) * p->Cout + co] = src[((size_t)co * p->K + k) * p->Cin + ci];
    p->bq = (const int32_t*)b->data;
    p->qm = (int32_t*)malloc(sizeof(int32_t) * (size_t)p->Cout);
    p->qs = (int*)malloc(sizeof(int) * (size_t)p->Cout);
    for (int co = 0; co < p->Cout; ++co) {
      const float fs = w->scale[w->nscale > 1 ? co : 0];
      const double eff = (double)x->scale[0] * (double)fs / (double)y->scale[0];
      lo_quantize_multiplier(eff, &p->qm[co], &p->qs[co]);
    }
    p->in_off = -(int32_t)x->zero_point[0];
    p->out_off = (int32_t)y->zero_point[0];
    p->scratch = (int32_t*)malloc(sizeof(int32_t) * (size_t)p->Tout * p->Cout);
  }
  return 0;
}

/* ---------------------------------------------------------------- op evaluation ---- */

static void eval_conv_f32(const op_prep* p, const float* x, float* y) {
  float acc[512];
  for (int t = 0; t < p->Tout; ++t)
    for (int g = 0; g < p->groups; ++g) {
      for (int c = 0; c < p->CoutG; ++c) acc[c] = 0.0f;
      for (int k = 0; k < p->K; ++k) {
        const float* xr = x + (size_t)(t * p->stride + k * p->dil) * p->Cin + (size_t)g * p->CinG;
        const float* wk = p->wf + ((size_t)g * p->K + k) * p->CinG * p->CoutG;
        for (int ci = 0; ci < p->CinG; ++ci) {
          const float xv = xr[ci];
          const float* w = wk + (size_t)ci * p->CoutG;
          for (int c = 0; c < p->CoutG; ++c) acc[c] = fmaf(xv, w[c], acc[c]);
        }
      }
      float* yo = y + (size_t)t * p->Cout + (size_t)g * p->CoutG;
      const float* b = p->bf + (size_t)g * p->CoutG;
      for (int c = 0; c < p->CoutG; ++c) yo[c] = acc[c] + b[c];
    }
}

static void eval_conv_i8(const op_prep* p, const int8_t* x, int8_t* y) {
  int32_t acc[512];
  for (int t = 0; t < p->Tout; ++t)
    for (int g = 0; g < p->groups; ++g) {
      for (int c = 0; c < p->CoutG; ++c) acc[c] = 0;
      for (int k = 0; k < p->K; ++k) {
        const int8_t* xr = x + (size_t)(t * p->stride + k * p->dil) * p->Cin + (size_t)g * p->CinG;
        const int8_t* wk = p->wq + ((size_t)g * p->K + k) * p->CinG * p->CoutG;
        for (int ci = 0; ci < p->CinG; ++ci) {
          const int32_t xv = (int32_t)xr[ci] + p->in_off;
          const int8_t* w = wk + (size_t)ci * p->CoutG;
          for (int c = 0; c < p->CoutG; ++c) acc[c] += xv * (int32_t)w[c];
        }
      }
      for (int c = 0; c < p->CoutG; ++c) {
        const int co = g * p->CoutG + c;
        int32_t a = acc[c] + p->bq[co];
        a = lo_mbqm(a, p->qm[co], p->qs[co]) + p->out_off;
        y[(size_t)t * p->Cout + co] = (int8_t)clamp_i8(a);
      }
    }
}

static void eval_dw_f32(const op_prep* p, const float* x, float* y) {
  for (int t = 0; t < p->Tout; ++t)
    for (int c = 0; c < p->Cout; ++c) {
      float acc = 0.0f;
      for (int k = 0; k < p->K; ++k) acc = fmaf(x[(size_t)(t + k * p->dil) * p->Cin + c], p->wf[(size_t)k * p->Cin + c], acc);
      y[(size_t)t * p->Cout + c] = acc + p->bf[c];
    }
}
static void eval_dw_i8(const op_prep* p, const int8_t* x, int8_t* y) {
  for (int t = 0; t < p->Tout; ++t)
    for (int c = 0; c < p->Cout; ++c) {
      int32_t acc = 0;
      for (int k = 0; k < p->K; ++k)
        acc += ((int32_t)x[(size_t)(t + k * p->dil) * p->Cin + c] + p->in_off) * (int32_t)p->wq[(size_t)k * p->Cin + c];
      acc += p->bq[c];
      acc = lo_mbqm(acc, p->qm[c], p->qs[c]) + p->out_off;
      y[(size_t)t * p->Cout + c] = (int8_t)clamp_i8(acc);
    }
}

/* reference/transpose_conv.h: scatter; per output element the order is (t_in ascending, cin ascending) */
static void eval_tconv_f32(const op_prep* p, const float* x, float* y) {
  const size_t ny = (size_t)p->Tout * p->Cout;
  for (size_t i = 0; i < ny; ++i) y[i] = 0.0f;
  for (int ti = 0; ti < p->Tin; ++ti)
    for (int ci = 0; ci < p->Cin; ++ci) {
      const float xv = x[(size_t)ti * p->Cin + ci];
      for (int k = 0; k < p->K; ++k) {
        float* yo = y + (size_t)(ti * p->stride + k) * p->Cout;
        const float* w = p->wf + ((size_t)k * p->Cin + ci) * p->Cout;
        for (int co = 0; co < p->Cout; ++co) yo[co] = fmaf(xv, w[co], yo[co]);
      }
    }
  for (int t = 0; t < p->Tout; ++t)
    for (int co = 0; co < p->Cout; ++co) y[(size_t)t * p->Cout + co] = y[(size_t)t * p->Cout + co] + p->bf[co];
}
static void eval_tconv_i8(const op_prep* p, const int8_t* x, int8_t* y) {
  const size_t ny = (size_t)p->Tout * p->Cout;
  int32_t* s = p->scratch;
  for (size_t i = 0; i < ny; ++i) s[i] = 0;
  for (int ti = 0; ti < p->Tin; ++ti)
    for (int ci = 0; ci < p->Cin; ++ci) {
      const int32_t xv = (int32_t)x[(size_t)ti * p->Cin + ci] + p->in_off;
      for (int k = 0; k < p->K; ++k) {
        int32_t* so = s + (size_t)(ti * p->stride + k) * p->Cout;
        const int8_t* w = p->wq + ((size_t)k * p->Cin + ci) * p->Cout;
        for (int co = 0; co < p->Cout; ++co) so[co] += xv * (int32_t)w[co];
      }
    }
  for (int t = 0; t < p->Tout; ++t)
    for (int co = 0; co < p->Cout; ++co) {
      int32_t a = s[(size_t)t * p->Cout + co] + p->bq[co];
      a = lo_mbqm(a, p->qm[co], p->qs[co]) + p->out_off;
      y[(size_t)t * p->Cout + co] = (int8_t)clamp_i8(a);
    }
}

static int run_op(lo_net* n, int oi) {
  const tfl_op* op = &n->sg->ops[oi];
  const tfl_tensor* T = n->sg->tensors;
  op_prep* p = &n->prep[oi];
  switch (op->code) {
    case OP_CALL_ONCE: case OP_VAR_HANDLE: return 0;
    case OP_READ_VARIABLE: {
      const lo_var* v = &n->vars[n->var_of[op->in[0]]];
      if (!v->data || v->count != T[op->out[0]].count) return -1;
      memcpy(tbuf(n, op->out[0]), v->data, v->count * sizeof(float));
      return 0;
    }
    case OP_ASSIGN_VARIABLE: {
      lo_var* v = &n->vars[n->var_of[op->in[0]]];
      const tfl_tensor* s = &T[op->in[1]];
      if (s->type != TFL_F32 || v->count != s->count) return -1;
      memcpy(v->data, tdata(n, op->in[1]), v->count * sizeof(float));
      return 0;
    }
    case OP_RESHAPE: {
      const tfl_tensor* s = &T[op->in[0]];
      memcpy(tbuf(n, op->out[0]), tdata(n, op->in[0]), s->count * (size_t)esize(s->type));
      return 0;
    }
    case OP_CONCATENATION: {
      const tfl_tensor* y = &T[op->out[0]];
      int axis = tfl_opt_i32(n->m, op, 0, 0);       /* ConcatenationOptions{0 axis, 1 act} */
      if (axis < 0) axis += y->ndim;
      size_t outer = 1, es = (size_t)esize(y->type);
      for (int d = 0; d < axis; ++d) outer *= (size_t)y->shape[d];
      size_t yrow = 1;
      for (int d = axis; d < y->ndim; ++d) yrow *= (size_t)y->shape[d];
      uint8_t* dst = (uint8_t*)tbuf(n, op->out[0]);
      size_t off = 0;
      for (int i = 0; i < op->nin; ++i) {
        const tfl_tensor* s = &T[op->in[i]];
        if (s->type != y->type) return -1;
        if (s->nscale && y->nscale && (s->scale[0] != y->scale[0] || s->zero_point[0] != y->zero_point[0])) return -1;
        size_t srow = 1;
        for (int d = axis; d < s->ndim; ++d) srow *= (size_t)s->shape[d];
        const uint8_t* src = (const uint8_t*)tdata(n, op->in[i]);
        for (size_t o = 0; o < outer; ++o) memcpy(dst + (o * yrow + off) * es, src + o * srow * es, srow * es);
        off += srow;
      }
      return off == yrow ? 0 : -1;
    }
    case OP_STRIDED_SLICE: {
      const tfl_tensor *x = &T[op->in[0]], *y = &T[op->out[0]];
      const int32_t* bg = (const int32_t*)T[op->in[1]].data;
      const int32_t* en = (const int32_t*)T[op->in[2]].data;
      const int32_t* st = (const int32_t*)T[op->in[3]].data;
      /* StridedSliceOptions{0 begin_mask, 1 end_mask, 2 ellipsis_mask, 3 new_axis_mask, 4 shrink_axis_mask} */
      const int bm = tfl_opt_i32(n->m, op, 0, 0), em = tfl_opt_i32(n->m, op, 1, 0);
      if (tfl_opt_i32(n->m, op, 2, 0) || tfl_opt_i32(n->m, op, 3, 0) || tfl_opt_i32(n->m, op, 4, 0)) return -1;
      if (x->ndim != 4 || !bg || !en || !st) return -1;
      int b[4], e[4];
      for (int d = 0; d < 4; ++d) {
        if (st[d] != 1) return -1;
        int dim = x->shape[d];
        int bb = (bm >> d) & 1 ? 0 : bg[d], ee = (em >> d) & 1 ? dim : en[d];
        if (bb < 0) bb += dim;
        if (ee < 0) ee += dim;
        if (bb < 0) bb = 0;
        if (ee > dim) ee = dim;
        b[d] = bb; e[d] = ee;
        if (e[d] - b[d] != y->shape[d]) return -1;
      }
      const size_t es = (size_t)esize(x->type);
      const uint8_t* src = (const uint8_t*)tdata(n, op->in[0]);
      uint8_t* dst = (uint8_t*)tbuf(n, op->out[0]);
      size_t o = 0;
      for (int i0 = b[0]; i0 < e[0]; ++i0)
        for (int i1 = b[1]; i1 < e[1]; ++i1)
          for (int i2 = b[2]; i2 < e[2]; ++i2) {
            const size_t base = (((size_t)i0 * x->shape[1] + i1) * x->shape[2] + i2) * x->shape[3] + b[3];
            const size_t len = (size_t)(e[3] - b[3]);
            memcpy(dst + o * es, src + base * es, len * es);
            o += len;
          }
      return 0;
    }
    case OP_SPLIT: {
      const tfl_tensor* x = &T[op->in[1]];
      int axis = *(const int32_t*)T[op->in[0]].data;
      if (axis < 0) axis += x->ndim;
      if (axis != x->ndim - 1) return -1;
      const size_t rows = x->count / (size_t)x->shape[axis], es = (size_t)esize(x->type);
      const int part = x->shape[axis] / op->nout;
      const uint8_t* src = (const uint8_t*)tdata(n, op->in[1]);
      for (int j = 0; j < op->nout; ++j) {
        uint8_t* dst = (uint8_t*)tbuf(n, op->out[j]);
        for (size_t r = 0; r < rows; ++r)
          memcpy(dst + r * (size_t)part * es, src + (r * (size_t)x->shape[axis] + (size_t)j * part) * es, (size_t)part * es);
      }
      return 0;
    }
    case OP_CONV_2D:
      if (T[op->in[0]].type == TFL_F32) eval_conv_f32(p, (const float*)tdata(n, op->in[0]), (float*)tbuf(n, op->out[0]));
      else eval_conv_i8(p, (const int8_t*)tdata(n, op->in[0]), (int8_t*)tbuf(n, op->out[0]));
      return 0;
    case OP_DEPTHWISE_CONV_2D:
      if (T[op->in[0]].type == TFL_F32) eval_dw_f32(p, (const float*)tdata(n, op->in[0]), (float*)tbuf(n, op->out[0]));
      else eval_dw_i8(p, (const int8_t*)tdata(n, op->in[0]), (int8_t*)tbuf(n, op->out[0]));
      return 0;
    case OP_TRANSPOSE_CONV:
      if (T[op->in[2]].type == TFL_F32) eval_tconv_f32(p, (const float*)tdata(n, op->in[2]), (float*)tbuf(n, op->out[0]));
      else eval_tconv_i8(p, (const int8_t*)tdata(n, op->in[2]), (int8_t*)tbuf(n, op->out[0]));
      return 0;
    case OP_LEAKY_RELU: {
      const tfl_tensor* x = &T[op->in[0]];
      if (x->type == TFL_F32) {
        /* reference/leaky_relu.h: val > 0 ? val : val * alpha */
        const float* s = (const float*)tdata(n, op->in[0]);
        float* d = (float*)tbuf(n, op->out[0]);
        for (size_t i = 0; i < x->count; ++i) d[i] = s[i] > 0.0f ? s[i] : s[i] * p->alpha;
      } else {
        /* reference/leaky_relu.h QuantizeLeakyRelu */
        const int8_t* s = (const int8_t*)tdata(n, op->in[0]);
        int8_t* d = (int8_t*)tbuf(n, op->out[0]);
        for (size_t i = 0; i < x->count; ++i) {
          const int32_t v = (int32_t)s[i] - p->in_off;   /* in_off holds the input zero point here */
          const int32_t u = p->out_off + (v >= 0 ? lo_mbqm(v, p->m1, p->s1) : lo_mbqm(v, p->m2, p->s2));
          d[i] = (int8_t)clamp_i8(u);
        }
      }
      return 0;
    }
    case OP_QUANTIZE: {
      /* reference/quantize.h AffineQuantize: round-half-away(val / scale) + zero_point, clamp */
      const tfl_tensor *x = &T[op->in[0]], *y = &T[op->out[0]];
      if (x->type != TFL_F32 || y->type != TFL_I8) return -1;
      const float scale = y->scale[0];
      const int32_t zp = (int32_t)y->zero_point[0];
      const float* s = (const float*)tdata(n, op->in[0]);
      int8_t* d = (int8_t*)tbuf(n, op->out[0]);
      for (size_t i = 0; i < x->count; ++i) d[i] = (int8_t)clamp_i8((int32_t)roundf(s[i] / scale) + zp);
      return 0;
    }
    case OP_DEQUANTIZE: {
      /* reference/dequantize.h: scale * (val - zero_point) */
      const tfl_tensor* x = &T[op->in[0]];
      if (x->type != TFL_I8) return -1;
      const float scale = x->scale[0];
      const int32_t zp = (int32_t)x->zero_point[0];
      const int8_t* s = (const int8_t*)tdata(n, op->in[0]);
      float* d = (float*)tbuf(n, op->out[0]);
      for (size_t i = 0; i < x->count; ++i) d[i] = scale * (float)((int32_t)s[i] - zp);
      return 0;
    }
    case OP_ADD: case OP_SUB: {
      const tfl_tensor *a = &T[op->in[0]], *b = &T[op->in[1]], *y = &T[op->out[0]];
      if (tfl_opt_i8(n->m, op, 0, 0) != 0) return -1;   /* fused activation: none */
      if (a->type == TFL_F32) {
        const float* pa = (const float*)tdata(n, op->in[0]);
        const float* pb = (const float*)tdata(n, op->in[1]);
        float* d = (float*)tbuf(n, op->out[0]);
        if (a->count != y->count || (y->count % b->count) != 0) return -1;
        /* b broadcasts over trailing dims ([C] against [1,T,1,C]) */
        if (op->code == OP_ADD) for (size_t i = 0; i < y->count; ++i) d[i] = pa[i] + pb[i % b->count];
        else for (size_t i = 0; i < y->count; ++i) d[i] = pa[i] - pb[i % b->count];
      } else if (a->type == TFL_I8 && op->code == OP_ADD) {
        /* reference/integer_ops/add.h AddElementwise */
        if (a->count != y->count || b->count != y->count) return -1;
        const int8_t* pa = (const int8_t*)tdata(n, op->in[0]);
        const int8_t* pb = (const int8_t*)tdata(n, op->in[1]);
        int8_t* d = (int8_t*)tbuf(n, op->out[0]);
        for (size_t i = 0; i < y->count; ++i) {
          const int32_t v1 = (p->in_off + pa[i]) * (1 << p->left_shift);
          const int32_t v2 = (p->in2_off + pb[i]) * (1 << p->left_shift);
          const int32_t s1 = lo_mbqm(v1, p->m1, p->s1);
          const int32_t s2 = lo_mbqm(v2, p->m2, p->s2);
          const int32_t r = lo_mbqm(s1 + s2, p->m3, p->s3) + p->out_off;
          d[i] = (int8_t)clamp_i8(r);
        }
      } else {
        return -1;
      }
      return 0;
    }
    default:
      fprintf(stderr, "lyra_oracle: unsupported op code %d at op %d\n", op->code, oi);
      return -1;
  }
}

/* ---------------------------------------------------------------- create / run ---- */

static int run_init_subgraph(lo_net* n, int sgi) {
  /* CALL_ONCE target: pairs of VAR_HANDLE(shared_name) + ASSIGN_VARIABLE(handle, constant) */
  const tfl_subgraph* sg = &n->m->sub[sgi];
  int* var_of = (int*)malloc(sizeof(int) * (size_t)sg->ntensors);
  for (int i = 0; i < sg->ntensors; ++i) var_of[i] = -1;
  int rc = 0;
  for (int i = 0; i < sg->nops && rc == 0; ++i) {
    const tfl_op* op = &sg->ops[i];
    if (op->code == OP_VAR_HANDLE) {
      const char* s; int len = tfl_opt_str(n->m, op, 1, &s);   /* VarHandleOptions{0 container, 1 shared_name} */
      var_of[op->out[0]] = add_var(n, s, len);
    } else if (op->code == OP_ASSIGN_VARIABLE) {
      const tfl_tensor* c = &sg->tensors[op->in[1]];
      const int v = var_of[op->in[0]];
      if (v < 0 || !c->data || c->type != TFL_F32) { rc = -1; break; }
      lo_var* var = &n->vars[v];
      free(var->data);
      var->count = c->count;
      var->data = (float*)malloc(c->count * sizeof(float));
      memcpy(var->data, c->data, c->count * sizeof(float));
    } else {
      rc = -1;
    }
  }
  free(var_of);
  return rc;
}

void lo_net_free(lo_net* n) {
  if (!n) return;
  if (n->sg) {
    for (int i = 0; i < n->sg->ntensors; ++i) if (n->buf) free(n->buf[i]);
    for (int i = 0; i < n->sg->nops; ++i) if (n->prep) {
      free(n->prep[i].wf); free(n->prep[i].wq); free(n->prep[i].qm); free(n->prep[i].qs); free(n->prep[i].scratch);
    }
  }
  for (int i = 0; i < n->nvars; ++i) free(n->vars[i].data);
  free(n->buf); free(n->var_of); free(n->prep);
  tfl_free(n->m);
  free(n);
}

int lo_net_reset(lo_net* n) {
  /* re-run the CALL_ONCE init subgraph(s): every state variable back to its (all-zero) constant */
  for (int i = 0; i < n->sg->nops; ++i)
    if (n->sg->ops[i].code == OP_CALL_ONCE)
      if (run_init_subgraph(n, tfl_opt_i32(n->m, &n->sg->ops[i], 0, 1)) != 0) return -1;  /* CallOnceOptions{0 init_subgraph_index} */
  return 0;
}

lo_net* lo_net_create(const char* tflite_path) {
  tfl_model* m = tfl_load(tflite_path);
  if (!m) return NULL;
  lo_net* n = (lo_net*)calloc(1, sizeof(*n));
  n->m = m;
  int sgi = tfl_signature_subgraph(m, "serving_default");
  if (sgi < 0) sgi = 0;
  n->sg = &m->sub[sgi];
  const tfl_subgraph* sg = n->sg;
  n->buf = (void**)calloc((size_t)sg->ntensors, sizeof(void*));
  n->var_of = (int*)malloc(sizeof(int) * (size_t)sg->ntensors);
  n->prep = (op_prep*)calloc((size_t)sg->nops, sizeof(op_prep));
  for (int i = 0; i < sg->ntensors; ++i) {
    n->var_of[i] = -1;
    const tfl_tensor* t = &sg->tensors[i];
    if (!t->data && esize(t->type) > 0) n->buf[i] = calloc(t->count ? t->count : 1, (size_t)esize(t->type));
  }
  if (lo_net_reset(n) != 0) { lo_net_free(n); return NULL; }
  for (int i = 0; i < sg->nops; ++i) {
    const tfl_op* op = &sg->ops[i];
    const tfl_tensor* T = sg->tensors;
    op_prep* p = &n->prep[i];
    int rc = 0;
    switch (op->code) {
      case OP_VAR_HANDLE: {
        const char* s; int len = tfl_opt_str(m, op, 1, &s);
        const int v = find_var(n, s, len);
        if (v < 0) rc = -1;
        n->var_of[op->out[0]] = v;
        break;
      }
      case OP_CONV_2D: rc = prep_conv(n, op, p); break;
      case OP_DEPTHWISE_CONV_2D: rc = prep_dw(n, op, p); break;
      case OP_TRANSPOSE_CONV: rc = prep_tconv(n, op, p); break;
      case OP_LEAKY_RELU: {
        const tfl_tensor *x = &T[op->in[0]], *y = &T[op->out[0]];
        p->alpha = tfl_opt_f32(m, op, 0, 0.0f);     /* LeakyReluOptions{0 alpha} */
        if (x->type == TFL_I8) {
          /* kernels/activations.cc LeakyReluPrepare: float expressions widened to double */
          const double alpha_mult = (double)(x->scale[0] * p->alpha / y->scale[0]);
          const double ident_mult = (double)(x->scale[0] / y->scale[0]);
          lo_quantize_multiplier(ident_mult, &p->m1, &p->s1);
          lo_quantize_multiplier(alpha_mult, &p->m2, &p->s2);
          p->in_off = (int32_t)x->zero_point[0];
          p->out_off = (int32_t)y->zero_point[0];
        }
        break;
      }
      case OP_ADD: {
        const tfl_tensor *a = &T[op->in[0]], *b = &T[op->in[1]], *y = &T[op->out[0]];
        if (a->type == TFL_I8) {
          /* kernels/add.cc Prepare, general 8-bit path */
          p->left_shift = 20;
          const float maxs = a->scale[0] > b->scale[0] ? a->scale[0] : b->scale[0];
          const double twice_max = (double)(2 * maxs);
          const double r1 = (double)a->scale[0] / twice_max;
          const double r2 = (double)b->scale[0] / twice_max;
          const double ro = twice_max / (double)((float)(1 << p->left_shift) * y->scale[0]);
          lo_quantize_multiplier(r1, &p->m1, &p->s1);
          lo_quantize_multiplier(r2, &p->m2, &p->s2);
          lo_quantize_multiplier(ro, &p->m3, &p->s3);
          p->in_off = -(int32_t)a->zero_point[0];
          p->in2_off = -(int32_t)b->zero_point[0];
          p->out_off = (int32_t)y->zero_point[0];
        }
        break;
      }
      default: break;
    }
    if (rc != 0) {
      fprintf(stderr, "lyra_oracle: cannot prepare op %d (code %d) of %s\n", i, op->code, tflite_path);
      lo_net_free(n);
      return NULL;
    }
  }
  return n;
}

int lo_net_invoke(lo_net* n, const float* in, int n_in, float* out, int n_out) {
  const tfl_subgraph* sg = n->sg;
  const tfl_tensor* ti = &sg->tensors[sg->inputs[0]];
  const tfl_tensor* to = &sg->tensors[sg->outputs[0]];
  if ((size_t)n_in != ti->count || (size_t)n_out != to->count) return -1;
  memcpy(n->buf[sg->inputs[0]], in, sizeof(float) * (size_t)n_in);
  for (int i = 0; i < sg->nops; ++i)
    if (run_op(n, i) != 0) { fprintf(stderr, "lyra_oracle: op %d failed\n", i); return -2; }
  memcpy(out, n->buf[sg->outputs[0]], sizeof(float) * (size_t)n_out);
  return 0;
}

int lo_net_num_tensors(const lo_net* n) { return n->sg->ntensors; }

int lo_net_tensor_info(const lo_net* n, int idx, int* type, int* count, float* scale, int* zero_point) {
  if (idx < 0 || idx >= n->sg->ntensors) return -1;
  const tfl_tensor* t = &n->sg->tensors[idx];
  *type = t->type; *count = (int)t->count;
  *scale = t->nscale ? t->scale[0] : 0.0f;
  *zero_point = t->nzp ? (int)t->zero_point[0] : 0;
  return 0;
}

int lo_net_read_tensor(const lo_net* n, int idx, void* dst, int max_bytes) {
  if (idx < 0 || idx >= n->sg->ntensors) return -1;
  const tfl_tensor* t = &n->sg->tensors[idx];
  const size_t nb = t->count * (size_t)esize(t->type);
  if (nb == 0 || nb > (size_t)max_bytes) return -1;
  memcpy(dst, tdata(n, idx), nb);
  return (int)nb;
}

int lo_net_num_vars(const lo_net* n) { return n->nvars; }
const char* lo_net_var_name(const lo_net* n, int v) { return v >= 0 && v < n->nvars ? n->vars[v].name : NULL; }
int lo_net_var_count(const lo_net* n, int v) { return v >= 0 && v < n->nvars ? (int)n->vars[v].count : -1; }
int lo_net_read_var(const lo_net* n, int v, float* dst, int max_count) {
  if (v < 0 || v >= n->nvars || (int)n->vars[v].count > max_count) return -1;
  memcpy(dst, n->vars[v].data, n->vars[v].count * sizeof(float));
  return (int)n->vars[v].count;
}
