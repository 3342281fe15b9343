// datagen/tpch_dbgen_gpu.cu -- the generator of datagen/tpch_dbgen.c as CUDA kernels writing Arrow columns
// straight into HBM.  Test / bench infrastructure, like its C twin: neither product nor oracle.
//
// Why it exists: BASELINE.json quotes its metric at SF100 (600 M lineitem rows, 60 GB of Arrow columns for Q1) and
// at SF100 PER GPU when scaling to 8 GPUs; the host generator takes minutes for that and the rows would then have to
// cross PCIe.  dbgen's streams are Lehmer generators with O(log n) skip-ahead and a fixed advance per order row, so an
// order is generated independently by one thread.  tests/test_gpu_datagen.py pins every column bit-exactly against the
// C generator (which reproduces the reference's golden snapshot at SF0.001).
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr long long MODULUS = 2147483647LL, MULT = 16807LL;
// stream ids / seeds / boundaries: see tpch_dbgen.c (only the order + lineitem streams are needed here)
enum { O_CLRK = 0, O_ODATE, L_QTY, L_DCNT, L_TAX, L_SHIP, L_SMODE, L_PKEY, L_SKEY, L_SDTE, L_CDTE, L_RDTE, L_RFLG, O_PRIO, O_CKEY, O_LCNT, N_ST };
__constant__ long long SEED0[N_ST] = {1171034773, 1066728069, 209208115, 554590007, 721958466, 1371272478, 675466456, 1808217256, 2095021727,
                                     1769349045, 904914315, 373135028, 717419739, 591449447, 851767375, 1434868289};
__constant__ int BOUND[N_ST] = {1, 1, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 1, 1, 1};

__device__ __forceinline__ long long nth_element(long long n, long long seed) {
  long long mult = MULT, z = seed;
  while (n > 0) {
    if (n & 1) z = (mult * z) % MODULUS;
    n >>= 1;
    mult = (mult * mult) % MODULUS;
  }
  return z;
}
struct Stream {
  long long v;
  __device__ __forceinline__ void init(int id, long long row0) { v = nth_element(row0 * (long long)BOUND[id], SEED0[id]); }
  __device__ __forceinline__ long long uniform(long long lo, long long hi) {
    v = (v * MULT) % MODULUS;
    const double range = (double)(hi - lo + 1);
    return lo + (long long)(((double)v / 2147483647.0) * range);
  }
};

constexpr int DATE32_1992_01_01 = 8035, O_ODATE_SPAN = 2557 - 151 - 1, CURRENT_IDX = 1263;
__device__ __forceinline__ long long sparse_key(long long i) { return ((i >> 3) << 5) | (i & 7); }
__device__ __forceinline__ long long retail_price(long long p) { return 90000 + ((p / 10) % 20001) + (p % 1000) * 100; }
__device__ __forceinline__ ulonglong2 dec128(long long v) { ulonglong2 w; w.x = (unsigned long long)v; w.y = (unsigned long long)(v >> 63); return w; }
__device__ __forceinline__ ulonglong2 char_view(unsigned char c) { ulonglong2 w; w.x = 1ull | ((unsigned long long)c << 32); w.y = 0; return w; }

__global__ void count_lines_kernel(long long first, long long n, int* lines) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    Stream s; s.init(O_LCNT, first + r);
    lines[r] = (int)s.uniform(1, 7);
  }
}

}  // namespace

struct TpchGpuOut {     // device pointers; null = column not wanted.  Arrow layouts: Int64, Int32/Date32, Decimal128 (16 B), Utf8View (16 B)
  long long* o_orderkey; long long* o_custkey; int* o_orderdate; int* o_shippriority; ulonglong2* o_totalprice; ulonglong2* o_orderstatus;
  long long* l_orderkey; long long* l_partkey; long long* l_suppkey; int* l_linenumber;
  ulonglong2* l_quantity; ulonglong2* l_extendedprice; ulonglong2* l_discount; ulonglong2* l_tax;
  ulonglong2* l_returnflag; ulonglong2* l_linestatus; int* l_shipdate; int* l_commitdate; int* l_receiptdate;
};

namespace {
__global__ void gen_kernel(long long n_part, long long n_supp, long long n_cust, long long first, long long n, const long long* __restrict__ offs, TpchGpuOut o) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    const long long row = first + r, idx = row + 1;
    Stream ckey, odate, lcnt, qty, dcnt, tax, pkey, skey, sdte, cdte, rdte, rflg;
    ckey.init(O_CKEY, row); odate.init(O_ODATE, row); lcnt.init(O_LCNT, row);
    qty.init(L_QTY, row); dcnt.init(L_DCNT, row); tax.init(L_TAX, row); pkey.init(L_PKEY, row); skey.init(L_SKEY, row);
    sdte.init(L_SDTE, row); cdte.init(L_CDTE, row); rdte.init(L_RDTE, row); rflg.init(L_RFLG, row);
    const long long okey = sparse_key(idx);
    long long ck = ckey.uniform(1, n_cust);
    int delta = 1;
    while (ck % 3 == 0) { ck += delta; if (ck > n_cust) ck = n_cust; delta = -delta; }
    const long long od = odate.uniform(0, O_ODATE_SPAN);
    const int lines = (int)lcnt.uniform(1, 7);
    long long total = 0; int ocnt = 0;
    long long nl = offs[r];
    for (int l = 0; l < lines; ++l, ++nl) {
      const long long q = qty.uniform(1, 50), d = dcnt.uniform(0, 10), t = tax.uniform(0, 8);
      const long long pk = pkey.uniform(1, n_part);
      const long long rp = retail_price(pk);
      const long long sn = skey.uniform(0, 3);
      const long long sk = (pk + sn * (n_supp / 4 + (pk - 1) / n_supp)) % n_supp + 1;
      const long long ep = rp * q;
      total += ((ep * (100 - d)) / 100) * (100 + t) / 100;
      const long long sd = sdte.uniform(1, 121) + od;
      const long long cd = cdte.uniform(30, 90) + od;
      const long long rd = rdte.uniform(1, 30) + sd;
      unsigned char rf = 'N';
      if (rd <= CURRENT_IDX) rf = (rflg.uniform(1, 2) == 1) ? 'R' : 'A';
      unsigned char ls = 'O';
      if (sd <= CURRENT_IDX) { ocnt++; ls = 'F'; }
      if (o.l_orderkey) o.l_orderkey[nl] = okey;
      if (o.l_partkey) o.l_partkey[nl] = pk;
      if (o.l_suppkey) o.l_suppkey[nl] = sk;
      if (o.l_linenumber) o.l_linenumber[nl] = l + 1;
      if (o.l_quantity) o.l_quantity[nl] = dec128(q * 100);
      if (o.l_extendedprice) o.l_extendedprice[nl] = dec128(ep);
      if (o.l_discount) o.l_discount[nl] = dec128(d);
      if (o.l_tax) o.l_tax[nl] = dec128(t);
      if (o.l_returnflag) o.l_returnflag[nl] = char_view(rf);
      if (o.l_linestatus) o.l_linestatus[nl] = char_view(ls);
      if (o.l_shipdate) o.l_shipdate[nl] = (int)(DATE32_1992_01_01 + sd);
      if (o.l_commitdate) o.l_commitdate[nl] = (int)(DATE32_1992_01_01 + cd);
      if (o.l_receiptdate) o.l_receiptdate[nl] = (int)(DATE32_1992_01_01 + rd);
    }
    if (o.o_orderkey) o.o_orderkey[r] = okey;
    if (o.o_custkey) o.o_custkey[r] = ck;
    if (o.o_orderdate) o.o_orderdate[r] = (int)(DATE32_1992_01_01 + od);
    if (o.o_shippriority) o.o_shippriority[r] = 0;
    if (o.o_totalprice) o.o_totalprice[r] = dec128(total);
    if (o.o_orderstatus) o.o_orderstatus[r] = char_view(ocnt == 0 ? 'O' : (ocnt == lines ? 'F' : 'P'));
  }
}
}  // namespace

static const long long kMaxGrid = 132 * 16;      // grid-stride launches: 16 CTAs on each of an H100's 132 SMs

extern "C" {

// lines[r] = number of lineitems of order row first + r (device array of n ints)
int tpch_gpu_count_lines(long long first, long long n, int* lines, void* stream) {
  if (n <= 0) return 0;
  const int grid = (int)((n + 255) / 256 < kMaxGrid ? (n + 255) / 256 : kMaxGrid);
  count_lines_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(first, n, lines);
  return (int)cudaGetLastError();
}
// offs[r] = exclusive prefix of lines[] (device array of n int64); counts as in tpch_counts_get()
int tpch_gpu_generate(long long n_part, long long n_supp, long long n_cust, long long first, long long n, const long long* offs, const TpchGpuOut* out, void* stream) {
  if (n <= 0) return 0;
  const int grid = (int)((n + 127) / 128 < kMaxGrid ? (n + 127) / 128 : kMaxGrid);
  gen_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(n_part, n_supp, n_cust, first, n, offs, *out);
  return (int)cudaGetLastError();
}

}  // extern "C"
