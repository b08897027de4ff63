// synth.cu -- TPC-H-shaped / SIP-shaped synthetic columns generated directly in HBM.
// Bit-identical to oracle/tpch_gen.py: every value is a pure function of (table, column, row).
// One thread per row, fully coalesced stores; HBM-write bound (8 B/row at most).
#include "common.cuh"

namespace qk {
namespace {

constexpr uint64_t GOLDEN = 0x9E3779B97F4A7C15ULL;
constexpr uint64_t SEED_BASE = 0x5EED0000ULL;
enum { T_ORDERS = 1, T_LINEITEM = 2, T_CUSTOMER = 3, T_SUPPLIER = 4, T_TRADES = 8, T_QUOTES = 9 };
// hash stream ids (oracle/tpch_gen.py)
enum { C_CUSTKEY = 1, C_ORDERDATE, C_SUPPKEY, C_PARTKEY, C_QUANTITY, C_DISCOUNT, C_TAX, C_SHIPDELTA,
       C_COMMITDELTA, C_RECEIPTDELTA, C_RETFLAG, C_NATION, C_SEGMENT };
enum { C_TIME = 20, C_SYMBOL = 21, C_PAYLOAD0 = 22 };
constexpr int64_t DAY_1992_01_01 = 8035, ORDERDATE_SPAN = 2406, DAY_1995_06_17 = 9298;

__constant__ int8_t PAT_ORDER[28] = {0, 0, 0, 0, 1, 2, 2, 2, 2, 2, 2, 2, 3, 3, 3, 4, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6, 6, 6};
__constant__ int8_t PAT_LINE[28] = {1, 2, 3, 4, 1, 1, 2, 3, 4, 5, 6, 7, 1, 2, 3, 1, 2, 3, 4, 5, 1, 2, 1, 2, 3, 4, 5, 6};

__device__ __forceinline__ uint64_t hash_u64(int table, int col, int64_t idx) {
    uint64_t seed = mix64(SEED_BASE + (uint64_t)table * 256 + (uint64_t)col);
    return mix64(((uint64_t)idx + 1) * GOLDEN + seed);
}
__device__ __forceinline__ int64_t uniform(int table, int col, int64_t idx, uint64_t n) {
    return (int64_t)(((hash_u64(table, col, idx) >> 32) * n) >> 32);
}
__device__ __forceinline__ int64_t order_key(int64_t o) { return (o / 8) * 32 + (o % 8) + 1; }
__device__ __forceinline__ int64_t order_date(int64_t o) {
    return DAY_1992_01_01 + uniform(T_ORDERS, C_ORDERDATE, o, ORDERDATE_SPAN);
}

struct Sizes { int64_t n_orders, n_customer, n_supplier, n_part, n_symbols, gap; };

template <typename T>
__device__ __forceinline__ void put(void* out, int64_t k, T v) { ((T*)out)[k] = v; }

__global__ void k_synth(int table, int column, Sizes sz, int64_t lo, int64_t n, void* out) {
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = lo + k;
        if (table == T_ORDERS) {
            switch (column) {
                case 0: put<int64_t>(out, k, order_key(i)); break;
                case 1: {
                    int64_t n_valid = sz.n_customer - sz.n_customer / 3;
                    int64_t u = uniform(T_ORDERS, C_CUSTKEY, i, n_valid);
                    put<int64_t>(out, k, u + u / 2 + 1);
                } break;
                case 2: put<int32_t>(out, k, (int32_t)order_date(i)); break;
                default: put<int32_t>(out, k, 0); break;
            }
        } else if (table == T_LINEITEM) {
            const int r = (int)(i % 28);
            const int64_t oidx = ((i / 28) * 7 + PAT_ORDER[r]) % sz.n_orders;
            switch (column) {
                case 0: put<int64_t>(out, k, order_key(oidx)); break;
                case 1: put<int64_t>(out, k, 1 + uniform(T_LINEITEM, C_PARTKEY, i, sz.n_part)); break;
                case 2: put<int64_t>(out, k, 1 + uniform(T_LINEITEM, C_SUPPKEY, i, sz.n_supplier)); break;
                case 3: put<int32_t>(out, k, PAT_LINE[r]); break;
                case 4: put<double>(out, k, (double)(1 + uniform(T_LINEITEM, C_QUANTITY, i, 50))); break;
                case 5: {
                    int64_t q = 1 + uniform(T_LINEITEM, C_QUANTITY, i, 50);
                    int64_t pk = 1 + uniform(T_LINEITEM, C_PARTKEY, i, sz.n_part);
                    int64_t retail = 90000 + ((pk / 10) % 20001) + 100 * (pk % 1000);
                    put<double>(out, k, (double)(q * retail) / 100.0);
                } break;
                case 6: put<double>(out, k, (double)uniform(T_LINEITEM, C_DISCOUNT, i, 11) / 100.0); break;
                case 7: put<double>(out, k, (double)uniform(T_LINEITEM, C_TAX, i, 9) / 100.0); break;
                case 8: {
                    int64_t ship = order_date(oidx) + 1 + uniform(T_LINEITEM, C_SHIPDELTA, i, 121);
                    int64_t rcpt = ship + 1 + uniform(T_LINEITEM, C_RECEIPTDELTA, i, 30);
                    int64_t ra = uniform(T_LINEITEM, C_RETFLAG, i, 2);
                    put<uint8_t>(out, k, (uint8_t)(rcpt <= DAY_1995_06_17 ? ra * 2 : 1));
                } break;
                case 9: {
                    int64_t ship = order_date(oidx) + 1 + uniform(T_LINEITEM, C_SHIPDELTA, i, 121);
                    put<uint8_t>(out, k, (uint8_t)(ship > DAY_1995_06_17));
                } break;
                case 10: put<int32_t>(out, k, (int32_t)(order_date(oidx) + 1 + uniform(T_LINEITEM, C_SHIPDELTA, i, 121))); break;
                case 11: put<int32_t>(out, k, (int32_t)(order_date(oidx) + 30 + uniform(T_LINEITEM, C_COMMITDELTA, i, 61))); break;
                default: {
                    int64_t ship = order_date(oidx) + 1 + uniform(T_LINEITEM, C_SHIPDELTA, i, 121);
                    put<int32_t>(out, k, (int32_t)(ship + 1 + uniform(T_LINEITEM, C_RECEIPTDELTA, i, 30)));
                } break;
            }
        } else if (table == T_CUSTOMER) {
            switch (column) {
                case 0: put<int64_t>(out, k, i + 1); break;
                case 1: put<int64_t>(out, k, uniform(T_CUSTOMER, C_NATION, i, 25)); break;
                default: put<uint8_t>(out, k, (uint8_t)uniform(T_CUSTOMER, C_SEGMENT, i, 5)); break;
            }
        } else if (table == T_SUPPLIER) {
            switch (column) {
                case 0: put<int64_t>(out, k, i + 1); break;
                default: put<int64_t>(out, k, uniform(T_SUPPLIER, C_NATION, i, 25)); break;
            }
        } else {  // T_TRADES / T_QUOTES
            switch (column) {
                case 0: put<int64_t>(out, k, i * sz.gap + uniform(table, C_TIME, i, sz.gap)); break;
                case 1: {
                    double u = (double)uniform(table, C_SYMBOL, i, 1 << 24) / 16777216.0;
                    double s = u * u;
                    s = s * (double)sz.n_symbols;
                    int32_t sym = (int32_t)s;
                    if (sym > sz.n_symbols - 1) sym = (int32_t)sz.n_symbols - 1;
                    put<int32_t>(out, k, sym);
                } break;
                default: {
                    const int p = column - 2;
                    float v;
                    if (table == T_TRADES) {
                        v = p == 0 ? (float)uniform(table, C_PAYLOAD0, i, 10000) / 100.0f
                                   : (float)uniform(table, C_PAYLOAD0 + 1, i, 100000) / 100.0f;
                    } else {
                        v = p < 2 ? (float)uniform(table, C_PAYLOAD0 + p, i, 100000) / 100.0f
                                  : (float)uniform(table, C_PAYLOAD0 + p, i, 1000) / 10.0f;
                    }
                    put<float>(out, k, v);
                } break;
            }
        }
    }
}

int expected_dtype(int table, int column) {
    switch (table) {
        case T_ORDERS: return column <= 1 ? QK_I64 : QK_I32;
        case T_LINEITEM:
            if (column <= 2) return QK_I64;
            if (column == 3) return QK_I32;
            if (column <= 7) return QK_F64;
            if (column <= 9) return QK_U8;
            return QK_I32;
        case T_CUSTOMER: return column <= 1 ? QK_I64 : QK_U8;
        case T_SUPPLIER: return QK_I64;
        case T_TRADES: case T_QUOTES: return column == 0 ? QK_I64 : (column == 1 ? QK_I32 : QK_F32);
        default: return 0;
    }
}

}  // namespace
}  // namespace qk

extern "C" int qk_synth_column(int32_t table, int32_t column, const int64_t* sizes, int64_t row_lo,
                               int64_t nrows, void* out, int32_t out_dtype, void* stream) {
    using namespace qk;
    int dt = expected_dtype(table, column);
    if (!dt) QK_FAIL(QK_ERR_INVALID, "qk_synth_column: unknown table %d", table);
    if (dt != out_dtype) QK_FAIL(QK_ERR_INVALID, "qk_synth_column: table %d column %d is dtype %d, not %d", table, column, dt, out_dtype);
    if (nrows < 0 || !sizes || (nrows > 0 && !out)) QK_FAIL(QK_ERR_INVALID, "qk_synth_column: bad arguments");
    if (nrows == 0) return QK_OK;
    Sizes sz{sizes[0], sizes[1], sizes[2], sizes[3], sizes[4], sizes[5]};
    if (sz.n_orders <= 0 || sz.n_customer <= 0 || sz.n_supplier <= 0 || sz.n_part <= 0)
        QK_FAIL(QK_ERR_INVALID, "qk_synth_column: sizes must be positive");
    k_synth<<<grid_size(nrows, 32), 256, 0, (cudaStream_t)stream>>>(table, column, sz, row_lo, nrows, out);
    QK_LAUNCH_CHECK("k_synth");
    return QK_OK;
}
