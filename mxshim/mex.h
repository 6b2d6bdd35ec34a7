/* mex.h -- stand-alone re-implementation of the subset of the MATLAB/Octave MEX
 * C API that SeDuMi's MEX plugins use (SURVEY.md section 8b lists the ~25 entry
 * points; reference call sites e.g. blkchol.c:239-440, getada3.c:370-569).
 *
 * Purpose: (1) lets the reference C sources compile unmodified into oracle/_ref/
 * for parity testing; (2) lets the CUDA MEX stubs in sedumi_b200/mex/ be built and
 * driven from Python (ctypes) on a box that has neither MATLAB nor Octave.  On a
 * user's machine the same stubs compile against the real mex.h instead.
 *
 * Data model: column-major IEEE double dense matrices, CSC sparse matrices with
 * size_t jc/ir, and 1x1 structs with named fields -- nothing else is used by the
 * reference on this path.
 */
#ifndef MXSHIM_MEX_H
#define MXSHIM_MEX_H

#include <stddef.h>
#include <stdlib.h>
#include <stdbool.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef size_t    mwSize;
typedef size_t    mwIndex;
typedef ptrdiff_t mwSignedIndex;

typedef enum { mxREAL = 0, mxCOMPLEX = 1 } mxComplexity;

typedef enum {
  mxSHIM_DOUBLE = 0,   /* full real double matrix   */
  mxSHIM_SPARSE = 1,   /* CSC sparse real double    */
  mxSHIM_STRUCT = 2    /* 1x1 struct                */
} mxShimClass;

typedef struct mxArray_tag mxArray;

/* ---- creation / destruction ---- */
mxArray *mxCreateDoubleMatrix(mwSize m, mwSize n, mxComplexity flag);
mxArray *mxCreateDoubleScalar(double v);
mxArray *mxCreateSparse(mwSize m, mwSize n, mwSize nzmax, mxComplexity flag);
mxArray *mxCreateStructMatrix(mwSize m, mwSize n, int nfields, const char **fieldnames);
mxArray *mxDuplicateArray(const mxArray *a);
void     mxDestroyArray(mxArray *a);

/* ---- queries ---- */
double  *mxGetPr(const mxArray *a);
double  *mxGetPi(const mxArray *a);
mwIndex *mxGetJc(const mxArray *a);
mwIndex *mxGetIr(const mxArray *a);
mwSize   mxGetM(const mxArray *a);
mwSize   mxGetN(const mxArray *a);
mwSize   mxGetNzmax(const mxArray *a);
mwSize   mxGetNumberOfElements(const mxArray *a);
double   mxGetScalar(const mxArray *a);
bool     mxIsSparse(const mxArray *a);
bool     mxIsStruct(const mxArray *a);
bool     mxIsDouble(const mxArray *a);
bool     mxIsEmpty(const mxArray *a);
bool     mxIsComplex(const mxArray *a);

/* ---- struct fields (index must be 0: only 1x1 structs) ---- */
mxArray *mxGetField(const mxArray *a, mwIndex index, const char *fieldname);
void     mxSetField(mxArray *a, mwIndex index, const char *fieldname, mxArray *value);
int      mxAddField(mxArray *a, const char *fieldname);
int      mxGetNumberOfFields(const mxArray *a);
const char *mxGetFieldNameByNumber(const mxArray *a, int n);

/* ---- setters used by the reference to transplant buffers ---- */
void mxSetPr(mxArray *a, double *pr);
void mxSetIr(mxArray *a, mwIndex *ir);
void mxSetJc(mxArray *a, mwIndex *jc);
void mxSetM(mxArray *a, mwSize m);
void mxSetN(mxArray *a, mwSize n);
void mxSetNzmax(mxArray *a, mwSize nzmax);

/* ---- MEX allocator ---- */
void *mxCalloc(size_t n, size_t size);
void *mxMalloc(size_t n);
void *mxRealloc(void *p, size_t size);
void  mxFree(void *p);

/* ---- errors: mexErrMsgTxt does not return (longjmp to mxshim_call) ---- */
void mexErrMsgTxt(const char *msg);
void mexErrMsgIdAndTxt(const char *id, const char *fmt, ...);
void mexWarnMsgTxt(const char *msg);
int  mexPrintf(const char *fmt, ...);
void mxshim_assert_fail(const char *expr, const char *msg, const char *file, int line);

/* mxAssert: active only in debug builds (mex -g); release mex compiles it away. */
#if defined(MXSHIM_DEBUG)
#define mxAssert(expr, msg) \
  do { if (!(expr)) mxshim_assert_fail(#expr, (msg), __FILE__, __LINE__); } while (0)
#else
#define mxAssert(expr, msg) ((void)0)
#endif

/* Every plugin exports exactly this symbol (e.g. getada3.c:370, blkchol.c:239). */
void mexFunction(int nlhs, mxArray *plhs[], int nrhs, const mxArray *prhs[]);

/* ---- harness entry (not part of the MEX API) ----
 * Calls fn(nlhs,plhs,nrhs,prhs) under a setjmp guard.  Returns 0 on success,
 * 1 if the plugin raised mexErrMsgTxt / a failed mxAssert (message retrievable
 * with mxshim_last_error()). */
typedef void (*mxshim_mexfn)(int, mxArray **, int, const mxArray **);
int         mxshim_call(mxshim_mexfn fn, int nlhs, mxArray **plhs, int nrhs, const mxArray **prhs);
const char *mxshim_last_error(void);
int         mxshim_class(const mxArray *a);

#ifdef __cplusplus
}
#endif
#endif /* MXSHIM_MEX_H */
