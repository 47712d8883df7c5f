/* Empty stand-in: the reference dcn_v2_im2col_cuda.cu includes this header but uses none of its contents
 * (see oracle/build_dcn_ref.py). */
