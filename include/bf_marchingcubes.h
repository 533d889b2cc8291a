/*
 * bf_marchingcubes.h -- C-ABI of the iso-surface extraction of the hashed TSDF (SURVEY.md section 8f, row N4, second half): the triangle mesh the
 * reference saves at the end of a scan (Ctrl+9 / s_generateMeshDir), and the mesh clean-up and PLY writer behind CUDAMarchingCubesHashSDF::saveMesh.
 *
 * Reference interface this replaces (FL/ = /root/reference/FriedLiver/Source/, mLib = /root/reference/external/mLib/include):
 *   extern "C" resetMarchingCubesCUDA, extractIsoSurfaceCUDA                  FL/DepthSensing/CUDAMarchingCubesHashSDF.cpp:7-11 (kernels: CUDAMarchingCubesSDF.cu:10-52)
 *   struct MarchingCubesParams, MarchingCubesData (Vertex, Triangle)          FL/DepthSensing/MarchingCubesSDFUtil.h:9-23, 27-287
 *   MarchingCubesData::extractIsoSurfaceAtPosition, vertexInterp              FL/DepthSensing/MarchingCubesSDFUtil.h:121-242
 *   class CUDAMarchingCubesHashSDF (create, extractIsoSurface, copyTrianglesToCPU, saveMesh)   FL/DepthSensing/CUDAMarchingCubesHashSDF.{h,cpp}
 *   MeshData::mergeCloseVertices(thresh, approx = true), removeDuplicateFaces, removeDegeneratedFaces   mLib core-mesh/meshData.cpp:40-100, 200-300
 *   MeshIO::saveToPLY                                                         mLib core-mesh/meshIO.cpp:556-640
 * Out of this header's scope: the chunk-grid overload of extractIsoSurface (FL/DepthSensing/CUDAMarchingCubesHashSDF.cpp:117-160) -- it walks the
 * host-streamed chunk grid, which BundleFusion runs with streaming off (SURVEY.md section 8: out of scope).
 *
 * The reference appends triangles with one atomicAdd each, so the ORDER of its triangle soup differs from run to run; the parity statement is on the
 * multiset of triangles (each with its three vertices in the reference's order).  Here a block's triangles are contiguous and ordered by voxel.
 *
 * A fixed triangle buffer drops what does not fit, as the reference's appendTriangle does.  For a model of any size: bfMarchingCubesCount counts
 * the triangles of every 512-slot chunk of the table on the device, bfMarchingCubesExtractRange extracts the blocks of a chunk range, and
 * bfMarchingCubesExtractIsoSurfaceWhole meshes the whole model through the class's buffer in parts cut between chunks.  The class's fixed path
 * keeps the count from before the clamp (bfMarchingCubesGetLastExtraction), so a loss is on record.
 */
#ifndef BF_MARCHINGCUBES_H
#define BF_MARCHINGCUBES_H

#include <stddef.h>
#include <stdint.h>

#include "bf_raycast.h"
#include "bf_tsdf.h"

#ifdef __cplusplus
extern "C" {
#endif

/* FL/DepthSensing/MarchingCubesSDFUtil.h:9-23 (64 bytes) */
typedef struct BFMarchingCubesParams {
    uint8_t  m_boxEnabled;                  /*  0  bool: only voxels whose centre lies in [m_minCorner, m_maxCorner] */
    uint8_t  m_pad[3];
    float    m_minCorner[3];                /*  4 */
    uint32_t m_maxNumTriangles;             /* 16  capacity of d_triangles */
    float    m_maxCorner[3];                /* 20 */
    uint32_t m_sdfBlockSize;                /* 32  8 */
    uint32_t m_hashNumBuckets;              /* 36 */
    uint32_t m_hashBucketSize;              /* 40 */
    float    m_threshMarchingCubes;         /* 44  largest jump between two corners of a cell (s_SDFMarchingCubeThreshFactor * voxel size) */
    float    m_threshMarchingCubes2;        /* 48  largest |sdf| of a corner */
    float    dummy[3];
} BFMarchingCubesParams;

typedef struct BFMarchingCubesVertex { float p[3]; float c[3]; } BFMarchingCubesVertex;                       /* position (world), colour / 255 */
typedef struct BFMarchingCubesTriangle { BFMarchingCubesVertex v0, v1, v2; } BFMarchingCubesTriangle;         /* 72 bytes */

/* FL/DepthSensing/MarchingCubesSDFUtil.h:281-286; device pointers, caller-owned (MarchingCubesData::allocate, :56-70) */
typedef struct BFMarchingCubesData {
    BFMarchingCubesParams*   d_params;      /* device copy of the parameters (MarchingCubesData::updateParams) */
    uint32_t*                d_numTriangles;
    BFMarchingCubesTriangle* d_triangles;   /* [m_maxNumTriangles] */
    uint8_t                  m_bIsOnGPU;
} BFMarchingCubesData;

/* ---- the reference's stubs, same names.  Errors print and exit(-1) like cutilSafeCall. ---- */
void resetMarchingCubesCUDA(BFMarchingCubesData* data);
/* reads the cell parameters from data->d_params (device) and the hash parameters last given to updateConstantHashParams, as the reference's kernel reads
 * *d_params and c_hashParams; rayCastData is not read (the reference passes it only for its member functions) and may be NULL */
void extractIsoSurfaceCUDA(const BFHashDataStruct* hashData, const BFRayCastData* rayCastData, const BFMarchingCubesParams* params, BFMarchingCubesData* data);

/* ---- bf* extension: explicit parameters, cudaError_t return codes, no host synchronisation ---- */
/* reset + extraction in one call: *d_numTriangles = min(triangles found, params->m_maxNumTriangles) when the stream reaches the end of the call.
 * Triangles past the capacity are dropped, and which ones survive depends on the order in which blocks reserve their ranges. */
int bfMarchingCubesExtract(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFMarchingCubesParams* params,
                           BFMarchingCubesTriangle* d_triangles, uint32_t* d_numTriangles);

/* ---- meshing a model of any size in parts ----
 * The table's slots are cut into chunks of BF_MC_CHUNK_SLOTS consecutive slots, ceil(4 * buckets / 512) of them; a chunk is what one CTA of the
 * extraction processes.  Every triangle comes from the cells of exactly one block, and every block from one slot, so chunk ranges that
 * partition the table partition the triangle multiset.  Neither call synchronises with the host; malformed calls return cudaErrorInvalidValue,
 * enqueue nothing and name the reason in bfGetLastErrorString. */
#define BF_MC_CHUNK_SLOTS 512
/* the count pass: the extraction's cell tests (and params' box), no triangle written and no global atomic.  d_chunkCounts[c] (device, one entry
 * per chunk) = triangles of the blocks in chunk c, written with a plain store by the one CTA that owns the chunk, so deterministic;
 * *d_total = their sum.  params->m_maxNumTriangles is not read. */
int bfMarchingCubesCount(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFMarchingCubesParams* params, uint32_t* d_chunkCounts,
                         unsigned long long* d_total);
/* reset + extraction of the blocks whose slots lie in chunks [chunkBegin, chunkEnd); neighbour blocks outside the range are still read for the
 * cells' samples.  *d_numTriangles as bfMarchingCubesExtract, whose launch the full range [0, chunks) is.  An empty range leaves *d_numTriangles = 0.
 * Refused: chunkEnd past the table, chunkBegin > chunkEnd, a NULL counter. */
int bfMarchingCubesExtractRange(const BFHashDataStruct* hashData, const BFHashParams* hashParams, const BFMarchingCubesParams* params, uint32_t chunkBegin,
                                uint32_t chunkEnd, BFMarchingCubesTriangle* d_triangles, uint32_t* d_numTriangles);

/* ---- host side: class CUDAMarchingCubesHashSDF ---- */
typedef struct BFMarchingCubes BFMarchingCubes;
int  bfMarchingCubesCreate(const BFMarchingCubesParams* params, BFMarchingCubes** out);        /* create(): device triangle buffer of m_maxNumTriangles */
void bfMarchingCubesDestroy(BFMarchingCubes* mc);
/* extractIsoSurface(hashData, hashParams, rayCastData, minCorner, maxCorner, boxEnabled) + copyTrianglesToCPU: the triangles are APPENDED to the host mesh buffer */
int  bfMarchingCubesExtractIsoSurface(BFMarchingCubes* mc, const BFHashDataStruct* hashData, const BFHashParams* hashParams, const float* minCorner, const float* maxCorner,
                                      int boxEnabled);
/* the whole mesh through the class's buffer, in as many parts as it takes (two or more host synchronisations):
 *   1. bfMarchingCubesCount, then the chunk counts read back (one synchronisation);
 *   2. if one chunk holds more triangles than the buffer (m_maxNumTriangles), the buffer is enlarged to that chunk's count and stays so;
 *   3. consecutive chunks are cut greedily into parts of at most m_maxNumTriangles triangles; each non-empty part is extracted
 *      (bfMarchingCubesExtractRange), copied back and appended to the host mesh buffer as bfMarchingCubesExtractIsoSurface appends (one
 *      synchronisation per part).
 * saveMesh then applies unchanged.  No triangle is dropped: trianglesExtracted == trianglesCounted. */
typedef struct BFMarchingCubesWholeInfo {
    uint64_t trianglesCounted;              /* the count pass's total */
    uint64_t trianglesExtracted;            /* the triangles the parts' extractions produced (appended to the mesh buffer) */
    uint32_t chunks;                        /* chunks of the table */
    uint32_t parts;                         /* non-empty parts extracted */
    uint32_t largestPart;                   /* triangles of the largest part */
    uint32_t bufferTriangles;               /* the buffer's capacity after the call */
    uint32_t bufferEnlarged;                /* 1: a chunk held more triangles than the buffer had room for */
    uint32_t hostSyncs;                     /* host synchronisations: 1 + parts */
} BFMarchingCubesWholeInfo;
int  bfMarchingCubesExtractIsoSurfaceWhole(BFMarchingCubes* mc, const BFHashDataStruct* hashData, const BFHashParams* hashParams, const float* minCorner,
                                           const float* maxCorner, int boxEnabled, BFMarchingCubesWholeInfo* info);
/* the last extraction of either call: *found = triangles its cells produced, *kept = triangles it appended to the mesh buffer.  found > kept
 * means a full buffer dropped found - kept triangles (bfMarchingCubesExtractIsoSurface; the whole-mesh call drops none). */
int  bfMarchingCubesGetLastExtraction(const BFMarchingCubes* mc, unsigned long long* found, unsigned long long* kept);
void bfMarchingCubesClearMeshBuffer(BFMarchingCubes* mc);
/* the host mesh buffer: triangle soup, three vertices per triangle; pointers stay valid until the next call on `mc` */
size_t bfMarchingCubesGetSoup(const BFMarchingCubes* mc, const float** positions /* [n][3] */, const float** colors /* [n][4], alpha 1 */);
/* saveMesh(filename, transform, overwriteExistingFile): index buffer, mergeCloseVertices(0.00001f, approx), removeDuplicateFaces, optional 4x4 row-major transform,
 * binary little-endian PLY; clears the mesh buffer.  With overwrite == 0 an existing file is kept and the name gets a numeric suffix, as in the reference;
 * actualPath (may be NULL) receives the name written. */
int  bfMarchingCubesSaveMesh(BFMarchingCubes* mc, const char* filename, const float* transform, int overwrite, char* actualPath, size_t actualPathCapacity);

/* ---- the mesh clean-up by itself (host memory; what saveMesh runs) ---- */
/* in: soup of numVertices vertices (positions [n][3], colours [n][4]) and numFaces index triples; out: merged vertices (in place, the first *numVerticesOut entries) and
 * faces (in place, the first *numFacesOut triples) -- mergeCloseVertices(thresh, true) then removeDuplicateFaces, in the reference's order of operations */
int  bfMeshMergeCloseVertices(float* positions, float* colors, size_t numVertices, uint32_t* faces, size_t numFaces, float thresh, size_t* numVerticesOut, size_t* numFacesOut);
int  bfMeshRemoveDuplicateFaces(uint32_t* faces, size_t numFaces, size_t* numFacesOut);
int  bfMeshSavePly(const char* filename, const float* positions, const float* colors /* [n][4] or NULL */, size_t numVertices, const uint32_t* faces, size_t numFaces);
/* saveMesh's transform (MeshData::applyTransform): p' = M * (p, 1) with M row-major 4x4, de-homogenised, in place on host positions [n][3] */
int  bfMeshApplyTransform(float* positions, size_t numVertices, const float* transform);

/* ---- the mesh clean-up on the device ----
 * bfMeshWeld takes a triangle soup in device memory in the extraction's layout (vertex i = soup vertex i, face t = (3t, 3t+1, 3t+2)) and writes
 * what bfMeshMergeCloseVertices(thresh) followed by bfMeshRemoveDuplicateFaces give on the same soup with colours (c, 1), bit for bit: merged
 * positions in first-occurrence order, their colours with w = 1, faces in their surviving order.  Vertices no face references are kept.
 * The result does not depend on thread scheduling.  It runs on the library stream (bfSetStream) and synchronises the host once per round of
 * the vertex merge plus once at the end (BFMeshWeldInfo.hostSyncs).  The caller owns the workspace (bfMeshWeldWorkspaceBytes, about
 * 90-150 bytes per triangle) and the outputs, sized for the worst case: positions [3T][3], colours [3T][4], faces [T][3].
 * Refused before anything is enqueued (cudaErrorInvalidValue, reason in bfGetLastErrorString): a NULL info; NULL pointers when T > 0; thresh
 * not finite or not > 0; 3T >= 2^31 (PLY indices are int); a workspace smaller than bfMeshWeldWorkspaceBytes(T).
 * Refused on the device: a position that is not finite, or whose cell index (p / thresh, rounded as the host rounds it) lies outside int32;
 * the call then returns cudaErrorInvalidValue with *info all zero and nothing written to the outputs. */
typedef struct BFMeshWeldInfo {
    uint64_t trianglesIn;                   /* T */
    uint64_t verticesOut;                   /* merged vertices written to positions / colours */
    uint64_t degenerateFaces;               /* faces with a repeated index after the merge (removeDegeneratedFaces) */
    uint64_t duplicateFaces;                /* non-degenerate faces whose vertex set an earlier face has (removeDuplicateFaces) */
    uint64_t facesOut;                      /* T - degenerateFaces - duplicateFaces */
    uint32_t cells;                         /* occupied cells of size thresh */
    uint32_t rounds;                        /* rounds of the vertex merge: 1 + the longest chain of cells that wait for an earlier neighbour */
    uint32_t hostSyncs;                     /* rounds + 1 */
} BFMeshWeldInfo;
size_t bfMeshWeldWorkspaceBytes(uint64_t numTriangles);     /* 0 when 3 * numTriangles >= 2^31 */
int  bfMeshWeld(const BFMarchingCubesTriangle* d_soup, uint64_t numTriangles, float thresh, void* d_workspace, size_t workspaceBytes,
                float* d_positions /* [3T][3] */, float* d_colors /* [3T][4] */, uint32_t* d_faces /* [T][3] */, BFMeshWeldInfo* info);

#ifdef __cplusplus
}
#endif
#endif /* BF_MARCHINGCUBES_H */
