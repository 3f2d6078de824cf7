// expr.cu — scalar expressions over record batches and tables: one launch of a register program.
//
// ExecuteScalarExpression (arrow/compute/exprs/exec.go:542-700) evaluates an expression tree (arrow/compute/
// expression.go) node by node: every inner call writes a whole column that the next call reads back.  The host
// compiler (host/compute.cc) turns a bound tree into the program of include/arrowgpu.h (ag_expr_program), and
// expr_eval_kernel runs it over every span of the input in one launch.  Every op calls the element functors of
// elem_ops.cuh, the same code the single-op kernels run, with the same slot rules: ScalarBinaryNotNull ops write 0
// under a null, ScalarBinary ops, comparisons and bitmap ops compute every slot.
//
// Layout: 256-thread blocks, 1024-row tiles; tiles start at span starts.  Each warp owns 128 consecutive rows of a
// tile (4 rows per lane, 4 validity / boolean words) and touches no other warp's rows, so the program runs without
// block barriers.  The registers live in dynamic shared memory: 8 B per row for values, 32-bit words for validity
// and for BOOL data.  An instruction is decoded once per warp per tile (warp-uniform), then applied to the warp's
// rows.  Columns are read straight from HBM by the LOAD instructions; the output register is stored once per tile
// (values as typed stores, bitmaps by atomicOr into words zeroed before the launch, since a tile's first row need not
// fall on a word boundary).
#include "common.cuh"
#include "elem_ops.cuh"
#include "host_stage.cuh"

#include <atomic>
#include <vector>

namespace ag {

namespace {

constexpr int kExprThreads = 256;
constexpr int kExprTile = 1024;
constexpr int kExprRegs = AG_EXPR_MAX_REGS;
constexpr int kExprWords = kExprTile / 32;
constexpr int kExprSmem = kExprRegs * kExprTile * 8 + 2 * kExprRegs * kExprWords * 4;

// One instruction as the kernel reads it: the ABI fields plus, for CAST, the check kind and the safe bounds of its
// input type (cast.cu's cast_io: 0 none, 1 integer range, 2 float -> integer round trip).
struct ExprIns {
  int op, type, out_type, dst, a, b, check;
  unsigned long long bits;   // CONST: the value; CAST kind 1: lo
  unsigned long long hi;     // CAST kind 1: hi
  int valid;                 // CONST
};
struct ExprParams {
  int n_instr, n_cols, out_reg, out_type;
  ExprIns ins[AG_EXPR_MAX_INSTR];
};
struct ExprSpan { long long n, first_tile, out_pos; };
struct ExprCol { const void* vals; const uint8_t* valid; long long off; };

template <typename F>
__device__ __forceinline__ void dev_visit_type(int type, F&& f) {
  switch (type) {
    case AG_TYPE_UINT8: f(TypeTag<uint8_t>{}); break;
    case AG_TYPE_INT8: f(TypeTag<int8_t>{}); break;
    case AG_TYPE_UINT16: f(TypeTag<uint16_t>{}); break;
    case AG_TYPE_INT16: f(TypeTag<int16_t>{}); break;
    case AG_TYPE_UINT32: f(TypeTag<uint32_t>{}); break;
    case AG_TYPE_INT32: f(TypeTag<int32_t>{}); break;
    case AG_TYPE_UINT64: f(TypeTag<unsigned long long>{}); break;
    case AG_TYPE_INT64: f(TypeTag<long long>{}); break;
    case AG_TYPE_FLOAT32: f(TypeTag<float>{}); break;
    case AG_TYPE_FLOAT64: f(TypeTag<double>{}); break;
    default: break;
  }
}
template <typename T> struct Storage { using type = T; };
template <> struct Storage<int8_t> { using type = uint8_t; };
template <> struct Storage<int16_t> { using type = uint16_t; };
template <> struct Storage<int32_t> { using type = uint32_t; };
template <> struct Storage<long long> { using type = unsigned long long; };

// The warp's view of one tile.
struct Tile {
  uint64_t* V;        // [reg][row]
  uint32_t* VW;       // [reg][word] validity
  uint32_t* BW;       // [reg][word] BOOL data
  int lane, rbase;    // rbase: the warp's first tile row
  int len;            // rows of the tile
  long long gbase;    // output row of tile row 0
  long long* bad;     // this lane's lowest failing output row
  __device__ __forceinline__ int row(int k) const { return rbase + k * 32 + lane; }
  __device__ __forceinline__ int word(int k) const { return (rbase >> 5) + k; }
  __device__ __forceinline__ uint32_t lenmask(int k) const {
    const int m = len - (rbase + k * 32);
    return m >= 32 ? 0xffffffffu : (m <= 0 ? 0u : ((1u << m) - 1u));
  }
  template <typename T> __device__ __forceinline__ T rd(int reg, int r) const { return *reinterpret_cast<const T*>(V + reg * kExprTile + r); }
  template <typename T> __device__ __forceinline__ void wr(int reg, int r, T v) const { *reinterpret_cast<T*>(V + reg * kExprTile + r) = v; }
  __device__ __forceinline__ uint32_t& vw(int reg, int k) const { return VW[reg * kExprWords + word(k)]; }
  __device__ __forceinline__ uint32_t& bw(int reg, int k) const { return BW[reg * kExprWords + word(k)]; }
  __device__ __forceinline__ void fail(int r) const {
    const long long g = gbase + r;
    if (r < len && g < *bad) *bad = g;
  }
};

// ScalarBinary over every slot (helpers.go:193-236): add / sub / mul / bit_wise_* run on the storage type, like
// launch_binary in elementwise.cu.
template <typename T, typename Op>
__device__ __forceinline__ void every_slot(const Tile& t, const ExprIns& in) {
  using S = typename Storage<T>::type;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = t.row(k);
    t.wr<S>(in.dst, r, Op::template apply<S>(t.rd<S>(in.a, r), t.rd<S>(in.b, r)));
  }
}

// The checked kernels of elementwise.cu: kNotNull rows are computed only where both operands are valid (0 elsewhere),
// otherwise every slot is computed (checked multiply, launch_checked_op).  A failing row lowers the error word.
template <typename T, typename Op, bool kNotNull>
__device__ __forceinline__ void checked_slots(const Tile& t, const ExprIns& in) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = t.row(k);
    const bool valid = !kNotNull || (((t.vw(in.a, k) & t.vw(in.b, k)) >> t.lane) & 1);
    T o = 0;
    if (valid) {
      bool bad;
      o = Op::apply(t.rd<T>(in.a, r), t.rd<T>(in.b, r), bad);
      if (bad) t.fail(r);
    }
    t.wr<T>(in.dst, r, o);
  }
}

template <typename T, typename Op>
__device__ __forceinline__ void unary_slots(const Tile& t, const ExprIns& in) {
#pragma unroll
  for (int k = 0; k < 4; ++k) { const int r = t.row(k); t.wr<T>(in.dst, r, Op::template apply<T, T>(t.rd<T>(in.a, r))); }
}

template <typename T, typename Cmp, bool kFlip>
__device__ __forceinline__ void compare_slots(const Tile& t, const ExprIns& in) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = t.row(k);
    const T x = t.rd<T>(in.a, r), y = t.rd<T>(in.b, r);
    const uint32_t bits = __ballot_sync(0xffffffffu, kFlip ? Cmp::template apply<T>(y, x) : Cmp::template apply<T>(x, y));
    if (t.lane == 0) t.bw(in.dst, k) = bits;
  }
}

template <typename I, typename O>
__device__ __forceinline__ void cast_slots(const Tile& t, const ExprIns& in) {
  const I lo = (I)in.bits, hi = (I)in.hi;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = t.row(k);
    const I v = t.rd<I>(in.a, r);
    const O o = cast_one<I, O>(v);
    const bool valid = (t.vw(in.a, k) >> t.lane) & 1;
    if (valid && ((in.check == 1 && cast_fails<I, O, 1>(v, o, lo, hi)) || (in.check == 2 && cast_fails<I, O, 2>(v, o, lo, hi)))) t.fail(r);
    t.wr<O>(in.dst, r, o);
  }
}

// Word phase of an instruction: lanes 0..3 own the warp's 4 words.  The __syncwarp orders it after the row phase, whose
// lanes may still read the words an in-place op (dst == a) rewrites here.
template <typename F>
__device__ __forceinline__ void words(const Tile& t, F&& f) {
  __syncwarp();
  if (t.lane < 4) f(t.lane);
}

__device__ __forceinline__ void exec_ins(const Tile& t, const ExprIns& in, const ExprCol* cols, long long row0, long long span_n) {
  const int lane = t.lane;
  switch (in.op) {
    case AG_EXPR_LOAD: {
      const ExprCol c = cols[in.a];
      const long long lo = c.off >> 3, hi = (c.off + span_n + 7) >> 3;
      if (in.out_type == AG_TYPE_BOOL) {
        words(t, [&](int k) { t.bw(in.dst, k) = bitmap_load32((const uint8_t*)c.vals, c.off + row0 + t.rbase + k * 32, lo, hi) & t.lenmask(k); });
      } else {
        dev_visit_type(in.out_type, [&](auto tag) {
          using T = typename decltype(tag)::type;
          T v[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) { const int r = t.row(k); v[k] = r < t.len ? __ldcs((const T*)c.vals + c.off + row0 + r) : T(0); }
#pragma unroll
          for (int k = 0; k < 4; ++k) t.wr<T>(in.dst, t.row(k), v[k]);
        });
      }
      words(t, [&](int k) {
        t.vw(in.dst, k) = (c.valid ? bitmap_load32(c.valid, c.off + row0 + t.rbase + k * 32, lo, hi) : 0xffffffffu) & t.lenmask(k);
      });
      break;
    }
    case AG_EXPR_CONST:
#pragma unroll
      for (int k = 0; k < 4; ++k) t.V[in.dst * kExprTile + t.row(k)] = in.bits;
      words(t, [&](int k) {
        t.bw(in.dst, k) = (in.bits & 0xff) ? 0xffffffffu : 0u;
        t.vw(in.dst, k) = in.valid ? t.lenmask(k) : 0u;
      });
      break;
    case AG_EXPR_NULL_OF:
#pragma unroll
      for (int k = 0; k < 4; ++k) t.V[in.dst * kExprTile + t.row(k)] = 0;
      words(t, [&](int k) { t.bw(in.dst, k) = 0; t.vw(in.dst, k) = 0; });
      break;
    case AG_EXPR_ADD: case AG_EXPR_SUB: case AG_EXPR_MUL: case AG_EXPR_BIT_AND: case AG_EXPR_BIT_OR: case AG_EXPR_BIT_XOR:
      dev_visit_type(in.type, [&](auto tag) {
        using T = typename decltype(tag)::type;
        switch (in.op) {
          case AG_EXPR_ADD: every_slot<T, OpAdd>(t, in); break;
          case AG_EXPR_SUB: every_slot<T, OpSub>(t, in); break;
          case AG_EXPR_MUL: every_slot<T, OpMul>(t, in); break;
          case AG_EXPR_BIT_AND: every_slot<T, OpBitAnd>(t, in); break;
          case AG_EXPR_BIT_OR: every_slot<T, OpBitOr>(t, in); break;
          default: every_slot<T, OpBitXor>(t, in); break;
        }
      });
      words(t, [&](int k) { t.vw(in.dst, k) = t.vw(in.a, k) & t.vw(in.b, k); });
      break;
    case AG_EXPR_ADD_CHECKED: case AG_EXPR_SUB_CHECKED: case AG_EXPR_MUL_CHECKED: case AG_EXPR_DIV: case AG_EXPR_DIV_CHECKED:
    case AG_EXPR_SHL: case AG_EXPR_SHR: case AG_EXPR_SHL_CHECKED: case AG_EXPR_SHR_CHECKED:
      dev_visit_type(in.type, [&](auto tag) {
        using T = typename decltype(tag)::type;
        if constexpr (std::is_floating_point<T>::value) {
          if (in.op == AG_EXPR_DIV) checked_slots<T, ChkFDiv<T, false>, true>(t, in);
          else checked_slots<T, ChkFDiv<T, true>, true>(t, in);
        } else {
          switch (in.op) {
            case AG_EXPR_ADD_CHECKED: checked_slots<T, ChkAdd<T>, true>(t, in); break;
            case AG_EXPR_SUB_CHECKED: checked_slots<T, ChkSub<T>, true>(t, in); break;
            case AG_EXPR_MUL_CHECKED: checked_slots<T, ChkMul<T>, false>(t, in); break;
            case AG_EXPR_DIV: case AG_EXPR_DIV_CHECKED: checked_slots<T, ChkDiv<T>, true>(t, in); break;
            case AG_EXPR_SHL: checked_slots<T, ChkShift<T, true, false>, true>(t, in); break;
            case AG_EXPR_SHR: checked_slots<T, ChkShift<T, false, false>, true>(t, in); break;
            case AG_EXPR_SHL_CHECKED: checked_slots<T, ChkShift<T, true, true>, true>(t, in); break;
            default: checked_slots<T, ChkShift<T, false, true>, true>(t, in); break;
          }
        }
      });
      words(t, [&](int k) { t.vw(in.dst, k) = t.vw(in.a, k) & t.vw(in.b, k); });
      break;
    case AG_EXPR_ABS: case AG_EXPR_NEG: case AG_EXPR_NEG_UNSIGNED_ZERO: case AG_EXPR_SIGN: case AG_EXPR_BIT_NOT:
      dev_visit_type(in.type, [&](auto tag) {
        using T = typename decltype(tag)::type;
        switch (in.op) {
          case AG_EXPR_ABS: unary_slots<T, UAbs>(t, in); break;
          case AG_EXPR_NEG: unary_slots<T, UNeg>(t, in); break;
          case AG_EXPR_NEG_UNSIGNED_ZERO: unary_slots<T, UNegChecked>(t, in); break;
          case AG_EXPR_SIGN: unary_slots<T, USign>(t, in); break;
          default: unary_slots<T, UBitNot>(t, in); break;
        }
      });
      words(t, [&](int k) { t.vw(in.dst, k) = t.vw(in.a, k); });
      break;
    case AG_EXPR_ABS_CHECKED: case AG_EXPR_NEG_CHECKED:
      // unary_checked_kernel: every slot, MinInt fails
      dev_visit_type(in.type, [&](auto tag) {
        using T = typename decltype(tag)::type;
        if constexpr (std::is_integral<T>::value && std::is_signed<T>::value) {
          using U = typename std::make_unsigned<T>::type;
          constexpr T tmin = (T)((U)1 << (sizeof(T) * 8 - 1));
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int r = t.row(k);
            const T v = t.rd<T>(in.a, r);
            if (v == tmin) t.fail(r);
            t.wr<T>(in.dst, r, in.op == AG_EXPR_ABS_CHECKED ? UAbs::apply<T, T>(v) : UNeg::apply<T, T>(v));
          }
        }
      });
      words(t, [&](int k) { t.vw(in.dst, k) = t.vw(in.a, k); });
      break;
    case AG_EXPR_EQ: case AG_EXPR_NE: case AG_EXPR_GT: case AG_EXPR_GE: case AG_EXPR_LT: case AG_EXPR_LE:
      dev_visit_type(in.type, [&](auto tag) {
        using T = typename decltype(tag)::type;
        using S = typename Storage<T>::type;   // == and != on the storage type, like compare_dev
        switch (in.op) {
          case AG_EXPR_EQ: compare_slots<S, CmpEq, false>(t, in); break;
          case AG_EXPR_NE: compare_slots<S, CmpNe, false>(t, in); break;
          case AG_EXPR_GT: compare_slots<T, CmpGt, false>(t, in); break;
          case AG_EXPR_GE: compare_slots<T, CmpGe, false>(t, in); break;
          case AG_EXPR_LT: compare_slots<T, CmpGt, true>(t, in); break;
          default: compare_slots<T, CmpGe, true>(t, in); break;
        }
      });
      __syncwarp();
      words(t, [&](int k) { t.vw(in.dst, k) = t.vw(in.a, k) & t.vw(in.b, k); });
      break;
    case AG_EXPR_AND: case AG_EXPR_OR: case AG_EXPR_XOR: case AG_EXPR_AND_NOT:
      words(t, [&](int k) {
        const uint32_t x = t.bw(in.a, k), y = t.bw(in.b, k);
        t.bw(in.dst, k) = in.op == AG_EXPR_AND ? word_op<W_AND>(x, y, 0, 0)
                        : in.op == AG_EXPR_OR ? word_op<W_OR>(x, y, 0, 0)
                        : in.op == AG_EXPR_XOR ? word_op<W_XOR>(x, y, 0, 0) : word_op<W_ANDNOT>(x, y, 0, 0);
        t.vw(in.dst, k) = t.vw(in.a, k) & t.vw(in.b, k);
      });
      break;
    case AG_EXPR_KLEENE_AND: case AG_EXPR_KLEENE_OR: case AG_EXPR_KLEENE_AND_NOT:
      words(t, [&](int k) {
        const uint32_t a = t.vw(in.a, k), b = t.bw(in.a, k), c = t.vw(in.b, k), d = t.bw(in.b, k);
        uint32_t v, o;
        if (in.op == AG_EXPR_KLEENE_AND) { v = word_op<W_KAND_V>(a, b, c, d); o = word_op<W_KAND_D>(a, b, c, d); }
        else if (in.op == AG_EXPR_KLEENE_OR) { v = word_op<W_KOR_V>(a, b, c, d); o = word_op<W_KOR_D>(a, b, c, d); }
        else { v = word_op<W_KANDNOT_V>(a, b, c, d); o = word_op<W_KANDNOT_D>(a, b, c, d); }
        t.vw(in.dst, k) = v & t.lenmask(k);
        t.bw(in.dst, k) = o;
      });
      break;
    case AG_EXPR_NOT:
      words(t, [&](int k) { t.bw(in.dst, k) = word_op<W_INVERT>(t.bw(in.a, k), 0, 0, 0); t.vw(in.dst, k) = t.vw(in.a, k); });
      break;
    case AG_EXPR_IS_NULL: case AG_EXPR_IS_NOT_NULL:
      words(t, [&](int k) {
        const uint32_t v = t.vw(in.a, k), m = t.lenmask(k);
        t.bw(in.dst, k) = in.op == AG_EXPR_IS_NULL ? (~v & m) : v;
        t.vw(in.dst, k) = m;
      });
      break;
    case AG_EXPR_IS_NAN:
      // isNanKernelExec: the != kernel with the input on both sides; integers are false; the output has no nulls
      dev_visit_type(in.type, [&](auto tag) {
        using T = typename decltype(tag)::type;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const T x = t.rd<T>(in.a, t.row(k));
          const uint32_t bits = __ballot_sync(0xffffffffu, std::is_floating_point<T>::value && CmpNe::apply<T>(x, x));
          if (lane == 0) t.bw(in.dst, k) = bits;
        }
      });
      __syncwarp();
      words(t, [&](int k) { t.vw(in.dst, k) = t.lenmask(k); });
      break;
    case AG_EXPR_CAST:
      dev_visit_type(in.type, [&](auto itag) {
        dev_visit_type(in.out_type, [&](auto otag) { cast_slots<typename decltype(itag)::type, typename decltype(otag)::type>(t, in); });
      });
      words(t, [&](int k) { t.vw(in.dst, k) = t.vw(in.a, k); });
      break;
    default: break;
  }
}

// OR the `bits` of 32 output rows starting at output row g into a zeroed bitmap.
__device__ __forceinline__ void or_bits(uint32_t* words_out, long long g, uint32_t bits) {
  if (!bits) return;
  const long long w = g >> 5;
  const int sh = (int)(g & 31);
  atomicOr(words_out + w, bits << sh);
  if (sh && (bits >> (32 - sh))) atomicOr(words_out + w + 1, bits >> (32 - sh));
}

__global__ void __launch_bounds__(kExprThreads, 3)
expr_eval_kernel(const __grid_constant__ ExprParams p, const ExprSpan* __restrict__ spans, int n_spans, long long total_tiles,
                 const ExprCol* __restrict__ cols, void* __restrict__ out, uint32_t* __restrict__ out_bits,
                 uint32_t* __restrict__ out_valid, long long* __restrict__ err) {
  extern __shared__ uint64_t smem[];
  long long my_bad = AG_NO_ERROR_POS;
  Tile t;
  t.V = smem;
  t.VW = reinterpret_cast<uint32_t*>(smem + kExprRegs * kExprTile);
  t.BW = t.VW + kExprRegs * kExprWords;
  t.lane = threadIdx.x & 31;
  t.rbase = (threadIdx.x >> 5) * 128;
  t.bad = &my_bad;
  for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int lo = 0, hi = n_spans - 1;   // last span with first_tile <= tile
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (spans[mid].first_tile <= tile) lo = mid; else hi = mid - 1;
    }
    const ExprSpan sp = spans[lo];
    const long long row0 = (tile - sp.first_tile) * kExprTile;
    t.len = (int)(sp.n - row0 < kExprTile ? sp.n - row0 : kExprTile);
    t.gbase = sp.out_pos + row0;
    const ExprCol* sc = cols + (long long)lo * p.n_cols;
    for (int pc = 0; pc < p.n_instr; ++pc) {
      exec_ins(t, p.ins[pc], sc, row0, sp.n);
      __syncwarp();
    }
    const int reg = p.out_reg;
    if (p.out_type == AG_TYPE_BOOL) {
      words(t, [&](int k) { or_bits(out_bits, t.gbase + t.rbase + k * 32, t.bw(reg, k) & t.lenmask(k)); });
    } else {
      dev_visit_type(p.out_type, [&](auto tag) {
        using T = typename decltype(tag)::type;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int r = t.row(k);
          if (r < t.len) __stcs((T*)out + t.gbase + r, t.rd<T>(reg, r));
        }
      });
    }
    if (out_valid) words(t, [&](int k) { or_bits(out_valid, t.gbase + t.rbase + k * 32, t.vw(reg, k) & t.lenmask(k)); });
    __syncwarp();
  }
  lower_error_row(my_bad, err);
}

bool is_value_type(int t) { return t == AG_TYPE_BOOL || type_width(t) != 0; }
bool is_int(int t) { return type_is_signed_int(t) || type_is_unsigned_int(t); }

// The checks of ag_eval_program[_dev]: every malformed program is AG_ERR_INVALID before any device work.  Register
// types are tracked through the program, so an operand must hold what the op takes.
ag_status expr_check(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, ExprParams* p) {
  if (!prog) AG_FAIL(AG_ERR_INVALID, "eval_program: NULL program");
  if (prog->n_instr < 1 || prog->n_instr > AG_EXPR_MAX_INSTR || !prog->instr)
    AG_FAIL(AG_ERR_INVALID, "eval_program: %d instructions (1 to %d)", prog->n_instr, AG_EXPR_MAX_INSTR);
  if (prog->n_cols < 0 || prog->n_cols > AG_EXPR_MAX_COLS || (prog->n_cols > 0 && !prog->col_types))
    AG_FAIL(AG_ERR_INVALID, "eval_program: %d columns (0 to %d)", prog->n_cols, AG_EXPR_MAX_COLS);
  for (int j = 0; j < prog->n_cols; ++j)
    if (!is_value_type(prog->col_types[j])) AG_FAIL(AG_ERR_INVALID, "eval_program: column %d has type %d", j, prog->col_types[j]);
  if (n_spans < 0 || (n_spans > 0 && prog->n_cols > 0 && !spans)) AG_FAIL(AG_ERR_INVALID, "eval_program: bad span table");
  int rt[kExprRegs];
  for (int r = 0; r < kExprRegs; ++r) rt[r] = -1;
  p->n_instr = prog->n_instr; p->n_cols = prog->n_cols;
  for (int i = 0; i < prog->n_instr; ++i) {
    const ag_expr_instr& s = prog->instr[i];
    ExprIns& d = p->ins[i];
    d = ExprIns{s.op, s.type, s.out_type, s.dst, s.a, s.b, 0, s.bits, 0, s.flags & 1};
    const auto reg_ok = [&](int r) { return r >= 0 && r < kExprRegs; };
    const auto typed = [&](int r, int t) { return reg_ok(r) && rt[r] == t; };
    if (!reg_ok(s.dst)) AG_FAIL(AG_ERR_INVALID, "eval_program: instruction %d writes register %d (0 to %d)", i, s.dst, kExprRegs - 1);
    bool ok = false;
    int out = s.type;
    switch (s.op) {
      case AG_EXPR_LOAD:
        ok = s.a >= 0 && s.a < prog->n_cols && prog->col_types[s.a] == s.type;
        break;
      case AG_EXPR_CONST: ok = is_value_type(s.type); break;
      case AG_EXPR_NULL_OF: ok = reg_ok(s.a) && rt[s.a] >= 0 && is_value_type(s.out_type); out = s.out_type; break;
      case AG_EXPR_ADD: case AG_EXPR_SUB: case AG_EXPR_MUL: case AG_EXPR_DIV: case AG_EXPR_DIV_CHECKED:
        ok = type_width(s.type) && typed(s.a, s.type) && typed(s.b, s.type);
        break;
      case AG_EXPR_ADD_CHECKED: case AG_EXPR_SUB_CHECKED: case AG_EXPR_MUL_CHECKED: case AG_EXPR_BIT_AND: case AG_EXPR_BIT_OR:
      case AG_EXPR_BIT_XOR: case AG_EXPR_SHL: case AG_EXPR_SHR: case AG_EXPR_SHL_CHECKED: case AG_EXPR_SHR_CHECKED:
        ok = is_int(s.type) && typed(s.a, s.type) && typed(s.b, s.type);
        break;
      case AG_EXPR_ABS: case AG_EXPR_NEG: case AG_EXPR_NEG_UNSIGNED_ZERO: case AG_EXPR_SIGN:
        ok = type_width(s.type) && typed(s.a, s.type);
        break;
      case AG_EXPR_BIT_NOT: ok = is_int(s.type) && typed(s.a, s.type); break;
      case AG_EXPR_ABS_CHECKED: case AG_EXPR_NEG_CHECKED: ok = type_is_signed_int(s.type) && typed(s.a, s.type); break;
      case AG_EXPR_EQ: case AG_EXPR_NE: case AG_EXPR_GT: case AG_EXPR_GE: case AG_EXPR_LT: case AG_EXPR_LE:
        ok = type_width(s.type) && typed(s.a, s.type) && typed(s.b, s.type);
        out = AG_TYPE_BOOL;
        break;
      case AG_EXPR_AND: case AG_EXPR_OR: case AG_EXPR_XOR: case AG_EXPR_AND_NOT:
      case AG_EXPR_KLEENE_AND: case AG_EXPR_KLEENE_OR: case AG_EXPR_KLEENE_AND_NOT:
        ok = s.type == AG_TYPE_BOOL && typed(s.a, s.type) && typed(s.b, s.type);
        break;
      case AG_EXPR_NOT: ok = s.type == AG_TYPE_BOOL && typed(s.a, s.type); break;
      case AG_EXPR_IS_NULL: case AG_EXPR_IS_NOT_NULL: ok = is_value_type(s.type) && typed(s.a, s.type); out = AG_TYPE_BOOL; break;
      case AG_EXPR_IS_NAN: ok = type_width(s.type) && typed(s.a, s.type); out = AG_TYPE_BOOL; break;
      case AG_EXPR_CAST:
        ok = type_width(s.type) && type_width(s.out_type) && typed(s.a, s.type);
        out = s.out_type;
        if (ok) {   // cast_io's choice of check, with the safe bounds of the input type
          const bool allow_int = (s.flags & AG_EXPR_ALLOW_INT_OVERFLOW) != 0, allow_float = (s.flags & AG_EXPR_ALLOW_FLOAT_TRUNCATE) != 0;
          visit_type(s.type, [&](auto itag) {
            return visit_type(s.out_type, [&](auto otag) {
              using I = typename decltype(itag)::type;
              using O = typename decltype(otag)::type;
              if (s.type == s.out_type) return AG_OK;
              if constexpr (!IsFloat<I>::v) {
                I lo = 0, hi = 0;
                if (!(IsFloat<O>::v ? allow_float : allow_int) && safe_bounds<I, O>(&lo, &hi)) {
                  d.check = 1; d.bits = (unsigned long long)lo; d.hi = (unsigned long long)hi;
                }
              } else if constexpr (!IsFloat<O>::v) {
                if (!allow_float) d.check = 2;
              }
              return AG_OK;
            }, [] { return AG_OK; });
          }, [] { return AG_OK; });
        }
        break;
      default: AG_FAIL(AG_ERR_INVALID, "eval_program: instruction %d has unknown op %d", i, s.op);
    }
    if (!ok) AG_FAIL(AG_ERR_INVALID, "eval_program: instruction %d (op %d): operands do not fit the op", i, s.op);
    if (s.op != AG_EXPR_CAST && s.op != AG_EXPR_NULL_OF && s.out_type != out)
      AG_FAIL(AG_ERR_INVALID, "eval_program: instruction %d (op %d): result type %d, the op gives %d", i, s.op, s.out_type, out);
    d.out_type = out;
    rt[s.dst] = out;
  }
  if (prog->out_reg < 0 || prog->out_reg >= kExprRegs || rt[prog->out_reg] < 0)
    AG_FAIL(AG_ERR_INVALID, "eval_program: output register %d holds no value", prog->out_reg);
  p->out_reg = prog->out_reg;
  p->out_type = rt[prog->out_reg];
  for (int64_t i = 0; i < n_spans; ++i) {
    const int64_t n = prog->n_cols > 0 ? spans[i * prog->n_cols].length : 0;
    for (int j = 0; j < prog->n_cols; ++j) {
      const ag_sort_chunk& c = spans[i * prog->n_cols + j];
      if (c.length != n || c.length < 0 || c.offset < 0) AG_FAIL(AG_ERR_INVALID, "eval_program: span %lld column %d: length %lld, offset %lld (span length %lld)",
                                                                  (long long)i, j, (long long)c.length, (long long)c.offset, (long long)n);
      if (c.length > 0 && !c.vals) AG_FAIL(AG_ERR_INVALID, "eval_program: span %lld column %d: NULL values", (long long)i, j);
    }
  }
  return AG_OK;
}

}  // namespace

ag_status eval_program_check(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans) {
  static ExprParams p;   // 8 KB: too large for the stack of every caller
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  return expr_check(prog, n_spans, spans, &p);
}

// n_spans spans of prog->n_cols columns each (host table of device pointers), output rows from 0.  A program with no
// columns has no rows.
ag_status eval_program_dev(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, void* out, uint8_t* out_valid,
                           int64_t* d_error_word, cudaStream_t st) {
  static ExprParams p;   // 8 KB: too large for the stack of every caller; guarded by the mutex below
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  AG_TRY(expr_check(prog, n_spans, spans, &p));
  std::vector<ExprSpan> sp;
  std::vector<ExprCol> cols;
  long long tiles = 0, rows = 0;
  for (int64_t i = 0; i < n_spans && prog->n_cols > 0; ++i) {
    const int64_t n = spans[i * prog->n_cols].length;
    if (n == 0) continue;
    sp.push_back(ExprSpan{n, tiles, rows});
    for (int j = 0; j < prog->n_cols; ++j) {
      const ag_sort_chunk& c = spans[i * prog->n_cols + j];
      cols.push_back(ExprCol{c.vals, c.valid, c.offset});
    }
    tiles += (n + kExprTile - 1) / kExprTile;
    rows += n;
  }
  if (rows == 0) return AG_OK;
  if (!out || !d_error_word) AG_FAIL(AG_ERR_INVALID, "eval_program: NULL output or error word");
  const bool bool_out = p.out_type == AG_TYPE_BOOL;
  if ((bool_out && (reinterpret_cast<uintptr_t>(out) & 3)) || (reinterpret_cast<uintptr_t>(out_valid) & 3) ||
      (!bool_out && (reinterpret_cast<uintptr_t>(out) & (type_width(p.out_type) - 1))))
    AG_FAIL(AG_ERR_INVALID, "eval_program: output not aligned (bitmaps: 4 bytes, values: their width)");
  const size_t words = (size_t)((rows + 31) / 32) * 4;
  if (bool_out) AG_CUDA_TRY(cudaMemsetAsync(out, 0, words, st));
  if (out_valid) AG_CUDA_TRY(cudaMemsetAsync(out_valid, 0, words, st));
  TableImage img(st);
  const size_t o_sp = img.add(sp), o_cols = img.add(cols);
  AG_TRY(img.upload("expression span table upload"));
  static std::atomic<unsigned> smem_done{0};
  AG_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(expr_eval_kernel), kExprSmem, &smem_done));
  int per_sm = 0;
  AG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, expr_eval_kernel, kExprThreads, kExprSmem));
  const long long cap = (long long)sm_count() * (per_sm > 0 ? per_sm : 1);
  const int grid = (int)(tiles < cap ? tiles : cap);
  expr_eval_kernel<<<grid, kExprThreads, kExprSmem, st>>>(p, img.at<ExprSpan>(o_sp), (int)sp.size(), tiles, img.at<ExprCol>(o_cols),
                                                          out, bool_out ? (uint32_t*)out : nullptr, (uint32_t*)out_valid,
                                                          (long long*)d_error_word);
  return check_launch("expr_eval_kernel");
}

}  // namespace ag

using namespace ag;

extern "C" ag_status ag_eval_program_dev(const ag_expr_program* prog, int64_t n_spans, const ag_sort_chunk* spans, void* out,
                                         uint8_t* out_valid, int64_t* d_error_word, ag_stream_t s) {
  AG_TRY(ensure_init());
  return eval_program_dev(prog, n_spans, spans, out, out_valid, d_error_word, resolve_stream(s));
}
