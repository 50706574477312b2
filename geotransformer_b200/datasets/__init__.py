"""Dataset metadata helpers of the benchmark evaluation."""
