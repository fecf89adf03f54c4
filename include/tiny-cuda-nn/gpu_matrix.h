/* tiny-cuda-nn/gpu_matrix.h -- GPUMatrix / GPUMatrixDynamic as applications use them (reference: gpu_matrix.h:60-520).
 * m() rows x n() columns; the DEFAULT layout is column-major, so a `GPUMatrix<float> batch(n_dims, batch_size)` is
 * sample-contiguous: element (dim, i) lives at data()[i * n_dims + dim] (gpu_matrix.h:226-228) -- exactly what the C ABI takes. */
#pragma once
#include "gpu_memory.h"

namespace tcnn {

template <typename T>
class GPUMatrixDynamic {
public:
	GPUMatrixDynamic() = default;
	GPUMatrixDynamic(uint32_t m, uint32_t n, MatrixLayout layout = CM) : m_rows{m}, m_cols{n}, m_layout{layout} {  /* owning */
		m_owned.resize((size_t)m * n);
		m_data = m_owned.data();
	}
	GPUMatrixDynamic(T* data, uint32_t m, uint32_t n, MatrixLayout layout = CM) : m_data{data}, m_rows{m}, m_cols{n}, m_layout{layout} {}  /* view */
	GPUMatrixDynamic(GPUMatrixDynamic&&) = default;
	GPUMatrixDynamic& operator=(GPUMatrixDynamic&&) = default;

	T* data() const { return m_data; }
	uint32_t m() const { return m_rows; }
	uint32_t rows() const { return m_rows; }
	uint32_t n() const { return m_cols; }
	uint32_t cols() const { return m_cols; }
	size_t n_elements() const { return (size_t)m_rows * m_cols; }
	size_t n_bytes() const { return n_elements() * sizeof(T); }
	MatrixLayout layout() const { return m_layout; }
	void memset(int value) { CUDA_CHECK_THROW(cudaMemset(m_data, value, n_bytes())); }
	void memset_async(cudaStream_t stream, int value) { CUDA_CHECK_THROW(cudaMemsetAsync(m_data, value, n_bytes(), stream)); }
	/* gpu_matrix.h:266-290: the elements in memory order, and a host-drawn fill (low + next_float() * (high - low), cast to T) */
	std::vector<T> to_cpu_vector() const {
		std::vector<T> v(n_elements());
		CUDA_CHECK_THROW(cudaMemcpy(v.data(), m_data, n_bytes(), cudaMemcpyDeviceToHost));
		return v;
	}
	template <typename RNG>
	void initialize_uniform(RNG& rnd, float low, float high) {
		const float scale = high - low;
		std::vector<T> v(n_elements());
		for (size_t i = 0; i < v.size(); ++i) v[i] = (T)(low + rnd.next_float() * scale);
		CUDA_CHECK_THROW(cudaMemcpy(m_data, v.data(), n_bytes(), cudaMemcpyHostToDevice));
	}

protected:
	T* m_data = nullptr;
	uint32_t m_rows = 0, m_cols = 0;
	MatrixLayout m_layout = CM;
	GPUMemory<T> m_owned;
};

template <typename T, MatrixLayout LAYOUT = MatrixLayout::ColumnMajor>
class GPUMatrix : public GPUMatrixDynamic<T> {
public:
	GPUMatrix() = default;
	GPUMatrix(uint32_t m, uint32_t n) : GPUMatrixDynamic<T>{m, n, LAYOUT} {}
	GPUMatrix(T* data, uint32_t m, uint32_t n) : GPUMatrixDynamic<T>{data, m, n, LAYOUT} {}
};

}  // namespace tcnn
