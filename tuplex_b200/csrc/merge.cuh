// merge.cuh — K9: in-order merge of resolved rows into a stage's normal output, on the device.
//
// Replaces ResolveTask::executeInOrder + emitNormalRows (tuplex/core/src/physical/ResolveTask.cc:878-1258, :300-375): the reference walks
// the normal partitions row by row and copies rows out until the running row number reaches the next resolved row's number
// (`while(_rowNumber != _currentRowNumber) writeRow(normal)`), i.e. an exception that was resolved returns to exactly the slot of the
// task's output stream it occupied (TransformTask.cc:764,885), an unresolved one leaves its slot empty.
// Closed form used here: exceptions sorted by row number r_0 < r_1 < ...; exception k had a_k = r_k - k normal rows before it. With the
// resolved subset m = 0 .. n_res - 1 (ascending): normal row j lands at j + #{m : a_m <= j}, resolved row m at a_m + m. One kernel
// writes the source selector of every output position, the gathers by selector (gather.cuh) then move each column once (columnar, coalesced
// on the output side).
#pragma once
#include <stdint.h>

namespace tplx {

constexpr uint32_t MERGE_B = 0x80000000u;  // selector flag: the row comes from the resolved block
// a selector never equals SEL_NONE (gather.cuh): tplx_gpu_result_merge_resolved refuses n_norm + n_res >= 2^31 - 1

// sel[n_norm + n_res]: j (normal row) or MERGE_B | m (resolved row)
__global__ void __launch_bounds__(256) merge_select_kernel(const uint64_t *__restrict__ a_res, uint64_t n_res, uint64_t n_norm, uint32_t *__restrict__ sel) {
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n_norm) {
        uint64_t lo = 0, hi = n_res;  // c = #{m : a_res[m] <= i}
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (a_res[mid] <= i) lo = mid + 1;
            else hi = mid;
        }
        sel[i + lo] = (uint32_t)i;
    } else if (i < n_norm + n_res) {
        const uint64_t m = i - n_norm;
        sel[a_res[m] + m] = MERGE_B | (uint32_t)m;
    }
}

}  // namespace tplx
